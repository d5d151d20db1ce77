// cv2.line(img, pt1, pt2, color, 1, LINE_8) on the device, shared by the M-LSD and OpenPose draw kernels: OpenCV's
// clipLine, then the pixels of its 8-connected LineIterator in closed form, one warp per line.
#pragma once
#include <cuda_runtime.h>

namespace pfd {

// OpenCV's clipLine(Size(W, H), pt1, pt2) in int64 (drawing.cpp): false when the segment misses the image.  A segment
// with both ends inside is left as it is.
__device__ inline bool clip_line(long long W, long long H, long long& x1, long long& y1, long long& x2, long long& y2) {
  const long long right = W - 1, bottom = H - 1;
  int c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8;
  int c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8;
  if ((c1 & c2) == 0 && (c1 | c2) != 0) {
    long long a;
    if (c1 & 12) {
      a = c1 < 8 ? 0 : bottom;
      x1 += (long long)__ddiv_rn(__dmul_rn((double)(a - y1), (double)(x2 - x1)), (double)(y2 - y1));
      y1 = a;
      c1 = (x1 < 0) + (x1 > right) * 2;
    }
    if (c2 & 12) {
      a = c2 < 8 ? 0 : bottom;
      x2 += (long long)__ddiv_rn(__dmul_rn((double)(a - y2), (double)(x2 - x1)), (double)(y2 - y1));
      y2 = a;
      c2 = (x2 < 0) + (x2 > right) * 2;
    }
    if ((c1 & c2) == 0 && (c1 | c2) != 0) {
      if (c1) {
        a = c1 == 1 ? 0 : right;
        y1 += (long long)__ddiv_rn(__dmul_rn((double)(a - x1), (double)(y2 - y1)), (double)(x2 - x1));
        x1 = a;
        c1 = 0;
      }
      if (c2) {
        a = c2 == 1 ? 0 : right;
        y2 += (long long)__ddiv_rn(__dmul_rn((double)(a - x2), (double)(y2 - y1)), (double)(x2 - x1));
        x2 = a;
        c2 = 0;
      }
    }
  }
  return (c1 | c2) == 0;
}

// put(x, y) for every pixel of cv2.line(..., 1, LINE_8) from (x1, y1) to (x2, y2) inside the W x H image, called by
// the 32 lanes of one warp.  After clipping and the left-to-right swap, LineIterator's pixel i (i = 0..D along the
// major axis, D >= d the axis lengths) has taken m_i = ceil((2 d i - D) / 2D) minor steps: its error term
// e_i = D - 2d(i + 1) + 2D m_i stays in [-2d, 2D - 2d), which fixes m_i.  Lane l visits i = l, l + 32, ...
template <typename Put>
__device__ __forceinline__ void for_each_line_pixel(long long W, long long H, long long x1, long long y1, long long x2,
                                                    long long y2, int lane, Put put) {
  if (!clip_line(W, H, x1, y1, x2, y2)) return;
  if (x2 < x1) {
    long long t = x1; x1 = x2; x2 = t;
    t = y1; y1 = y2; y2 = t;
  }
  const long long dx = x2 - x1, ady = y2 >= y1 ? y2 - y1 : y1 - y2;
  const long long sy = y2 >= y1 ? 1 : -1;
  const bool vert = ady > dx;
  const long long D = vert ? ady : dx, d = vert ? dx : ady;
  for (long long i = lane; i <= D; i += 32) {
    const long long a = 2 * d * i - D;
    const long long m = D == 0 ? 0 : (a >= 0 ? (a + 2 * D - 1) / (2 * D) : -((-a) / (2 * D)));
    const long long x = vert ? x1 + m : x1 + i, y = vert ? y1 + sy * i : y1 + sy * m;
    if (x >= 0 && x < W && y >= 0 && y < H) put(x, y);
  }
}

}  // namespace pfd
