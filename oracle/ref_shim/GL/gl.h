// oracle/ref_shim/GL/gl.h -- TEST INFRASTRUCTURE.  No-op stand-ins for the OpenGL calls lsd_slam_viewer/src/KeyFrameDisplay.cpp
// makes, so that the viewer's own source compiles and runs without a display.  glBufferData keeps a copy of the data, which makes
// refreshPC's vertex buffer observable (oracle/ref_viewer_driver.cpp reads it back).
#ifndef LSD_REF_SHIM_GL_H
#define LSD_REF_SHIM_GL_H

#include <cstddef>
#include <cstring>
#include <vector>

typedef unsigned int GLenum;
typedef unsigned int GLuint;
typedef int GLint;
typedef int GLsizei;
typedef float GLfloat;
typedef unsigned char GLboolean;
typedef void GLvoid;
typedef std::ptrdiff_t GLsizeiptr;

#define GL_LINES 0x0001
#define GL_POINTS 0x0000
#define GL_FLOAT 0x1406
#define GL_UNSIGNED_BYTE 0x1401
#define GL_BLEND 0x0BE2
#define GL_SRC_ALPHA 0x0302
#define GL_ONE_MINUS_SRC_ALPHA 0x0303
#define GL_LIGHTING 0x0B50
#define GL_LIGHT0 0x4000
#define GL_LIGHT1 0x4001
#define GL_AMBIENT 0x1200
#define GL_AMBIENT_AND_DIFFUSE 0x1602
#define GL_VERTEX_ARRAY 0x8074
#define GL_COLOR_ARRAY 0x8076
#define GL_ARRAY_BUFFER 0x8892
#define GL_STATIC_DRAW 0x88E4

namespace lsd_ref_shim_gl {
inline std::vector<unsigned char>& lastBuffer() { static std::vector<unsigned char> b; return b; }
inline GLuint& nextName() { static GLuint n = 0; return n; }
}

inline void glGenBuffers(GLsizei n, GLuint* ids) { for (GLsizei i = 0; i < n; i++) ids[i] = ++lsd_ref_shim_gl::nextName(); }
inline void glDeleteBuffers(GLsizei, const GLuint*) {}
inline void glBindBuffer(GLenum, GLuint) {}
inline void glBufferData(GLenum, GLsizeiptr size, const GLvoid* data, GLenum)
{
    std::vector<unsigned char>& b = lsd_ref_shim_gl::lastBuffer();
    b.resize((size_t)size);
    if (size) std::memcpy(b.data(), data, (size_t)size);
}
inline void glPushMatrix() {}
inline void glPopMatrix() {}
inline void glMultMatrixf(const GLfloat*) {}
inline void glColor3f(GLfloat, GLfloat, GLfloat) {}
inline void glLineWidth(GLfloat) {}
inline void glBegin(GLenum) {}
inline void glEnd() {}
inline void glVertex3f(GLfloat, GLfloat, GLfloat) {}
inline void glEnable(GLenum) {}
inline void glDisable(GLenum) {}
inline void glBlendFunc(GLenum, GLenum) {}
inline void glLightfv(GLenum, GLenum, const GLfloat*) {}
inline void glPointSize(GLfloat) {}
inline void glVertexPointer(GLint, GLenum, GLsizei, const GLvoid*) {}
inline void glColorPointer(GLint, GLenum, GLsizei, const GLvoid*) {}
inline void glEnableClientState(GLenum) {}
inline void glDisableClientState(GLenum) {}
inline void glDrawArrays(GLenum, GLint, GLsizei) {}

#endif
