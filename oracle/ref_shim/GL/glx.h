// oracle/ref_shim/GL/glx.h -- TEST INFRASTRUCTURE (see gl.h in this directory); KeyFrameDisplay.cpp calls nothing from GLX.
#pragma once
#include "gl.h"
