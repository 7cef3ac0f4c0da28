// Device helpers shared by the detectors that read uint8 images (superpoint.cu, sift.cu).
#pragma once
#include <stdint.h>

// cv2 COLOR_RGB2GRAY / COLOR_RGBA2GRAY for 8-bit: (9798 R + 19235 G + 3735 B + 2^14) >> 15   (utils/images.py:36-38).
// `p` points at one interleaved pixel of a 1-, 3- or 4-channel image.
__device__ __forceinline__ uint8_t b2_gray_u8(const uint8_t* p, int channels) {
  if (channels == 1) return p[0];
  const int v = 9798 * (int)p[0] + 19235 * (int)p[1] + 3735 * (int)p[2] + (1 << 14);
  return (uint8_t)(v >> 15);
}
