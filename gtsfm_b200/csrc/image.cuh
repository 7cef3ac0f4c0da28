// Device helpers shared by the detectors that read uint8 images (superpoint.cu, sift.cu, orb.cu).
#pragma once
#include <float.h>
#include <math.h>
#include <stdint.h>

// cv2 COLOR_RGB2GRAY / COLOR_RGBA2GRAY for 8-bit: (9798 R + 19235 G + 3735 B + 2^14) >> 15   (utils/images.py:36-38).
// `p` points at one interleaved pixel of a 1-, 3- or 4-channel image.
__device__ __forceinline__ uint8_t b2_gray_u8(const uint8_t* p, int channels) {
  if (channels == 1) return p[0];
  const int v = 9798 * (int)p[0] + 19235 * (int)p[1] + 3735 * (int)p[2] + (1 << 14);
  return (uint8_t)(v >> 15);
}

// cv2 hal::fastAtan2 (degrees, [0, 360)).  The products and sums round as written only where the including file is compiled
// with -fmad=false (orb.cu); elsewhere nvcc may contract them into FMAs.
__device__ __forceinline__ float b2_fast_atan2(float y, float x) {
  const float p1 = 0.9997878412794807f * (float)(180 / M_PI), p3 = -0.3258083974640975f * (float)(180 / M_PI);
  const float p5 = 0.1555786518463281f * (float)(180 / M_PI), p7 = -0.04432655554792128f * (float)(180 / M_PI);
  const float ax = fabsf(x), ay = fabsf(y);
  float a, c, c2;
  if (ax >= ay) {
    c = ay / (ax + (float)DBL_EPSILON);
    c2 = c * c;
    a = (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c;
  } else {
    c = ax / (ay + (float)DBL_EPSILON);
    c2 = c * c;
    a = 90.f - (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c;
  }
  if (x < 0) a = 180.f - a;
  if (y < 0) a = 360.f - a;
  return a;
}
