// oracle/ref_shim/QGLViewer/qglviewer.h -- TEST INFRASTRUCTURE.  What lsd_slam_viewer/src/KeyFrameDisplay.h takes from
// libQGLViewer: the OpenGL types (QGLViewer includes GL/gl.h) and Qt's global `uchar` (qglobal.h).
#pragma once
#include <GL/gl.h>
typedef unsigned char uchar;
