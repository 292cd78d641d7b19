// oracle/ref_shim/GL/glu.h -- TEST INFRASTRUCTURE (see gl.h in this directory); KeyFrameDisplay.cpp calls nothing from GLU.
#pragma once
#include "gl.h"
