// ref_photo_shim.cpp — the reference's PhotometricUndistorter (util/Undistort.cpp:20-214, UNMODIFIED) with a working image reader.  TEST INFRASTRUCTURE ONLY.
//
// oracle/Makefile's _ref/libsdvref.so links IOWrapper/ImageRW_dummy.cpp, whose readers return NULL, so its PhotometricUndistorter never becomes valid.
// oracle/gamma.mk links this file instead, with the reference's Undistort.cpp and settings.cpp only, into oracle/_ref/libsdvref_photo.so: the readers below
// take binary PGM (P5), 8-bit for readImageBW_8U and 16-bit (maxval > 255) for readImageBW_16U, each returning NULL for the other depth, as OpenCV's
// IMREAD_UNCHANGED reader the reference builds with returns no 16-bit image for an 8-bit file.  What it returns is stored in tests/golden/ref_pin_gamma.npz.
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>
#include "Eigen/Core"
#define private public                                     // G, GDepth, vignetteMapInv, valid
#include "util/Undistort.h"
#undef private
#include "util/settings.h"
#include "IOWrapper/ImageRW.h"

namespace sdv_loam { namespace IOWrap {
static bool read_pgm(const std::string& fn, int& w, int& h, int& maxv, std::vector<unsigned char>& body) {
  FILE* f = fopen(fn.c_str(), "rb"); if (!f) return false;
  char magic[3] = {0}; bool ok = fscanf(f, "%2s %d %d %d", magic, &w, &h, &maxv) == 4 && !strcmp(magic, "P5") && w > 0 && h > 0 && maxv > 0 && maxv < 65536 && fgetc(f) != EOF;
  if (ok) { body.resize((size_t)w*h*(maxv > 255 ? 2 : 1)); ok = fread(body.data(), 1, body.size(), f) == body.size(); }
  fclose(f); return ok;
}
MinimalImageB* readImageBW_8U(std::string filename) {
  int w, h, m; std::vector<unsigned char> b; if (!read_pgm(filename, w, h, m, b) || m > 255) return 0;
  MinimalImageB* img = new MinimalImageB(w, h); memcpy(img->data, b.data(), b.size()); return img;
}
MinimalImage<unsigned short>* readImageBW_16U(std::string filename) {
  int w, h, m; std::vector<unsigned char> b; if (!read_pgm(filename, w, h, m, b) || m <= 255) return 0;
  MinimalImage<unsigned short>* img = new MinimalImage<unsigned short>(w, h);
  for (size_t i = 0; i < (size_t)w*h; i++) img->data[i] = (unsigned short)((b[2*i] << 8) | b[2*i+1]);       // PGM samples are big-endian
  return img;
}
MinimalImageB3* readImageRGB_8U(std::string filename) { return 0; }
MinimalImageB* readStreamBW_8U(char* data, int numBytes) { return 0; }
void writeImage(std::string filename, MinimalImageB* img) {}
void writeImage(std::string filename, MinimalImageB3* img) {}
void writeImage(std::string filename, MinimalImageF* img) {}
void writeImage(std::string filename, MinimalImageF3* img) {}
} }

using namespace sdv_loam;
extern "C" {
// setting_photometricCalibration = pc, then the constructor; returns the object (valid or not)
void* ref_photo_create(const char* gamma_file, const char* vignette_file, int w, int h, int pc) {
  setting_photometricCalibration = pc;
  return new PhotometricUndistorter(gamma_file, "", vignette_file, w, h);
}
void ref_photo_destroy(void* p) { delete (PhotometricUndistorter*)p; }
// valid flag and GDepth; G (GDepth floats) when getG() is non-NULL; vignetteMapInv (w*h floats) when the constructor made it
int ref_photo_get(void* p, int* gdepth, float* G_out, float* vinv_out) {
  PhotometricUndistorter* u = (PhotometricUndistorter*)p; *gdepth = u->GDepth;
  if (u->getG() && G_out) memcpy(G_out, u->getG(), sizeof(float)*u->GDepth);
  if (u->vignetteMapInv && vinv_out) memcpy(vinv_out, u->vignetteMapInv, sizeof(float)*u->w*u->h);
  return u->valid ? 1 : 0;
}
// processFrame<unsigned char>(raw, exposure, factor) with setting_photometricCalibration = pc -> output->image
void ref_photo_process(void* p, const unsigned char* raw, float exposure, float factor, int pc, float* out) {
  PhotometricUndistorter* u = (PhotometricUndistorter*)p; setting_photometricCalibration = pc;
  std::vector<unsigned char> in(raw, raw + (size_t)u->w*u->h);
  u->processFrame<unsigned char>(in.data(), exposure, factor);
  memcpy(out, u->output->image, sizeof(float)*u->w*u->h);
}
}
