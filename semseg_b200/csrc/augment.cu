// Training-batch augmentation in one launch: tool/train.py:194-201's RandScale -> RandRotate -> RandomGaussianBlur ->
// RandomHorizontalFlip -> Crop -> ToTensor -> Normalize (util/transform.py) over decoded uint8 images, with the random
// parameters drawn on the host (semseg_b200/augment.py) and handed over in a per-sample descriptor table.
//
// CTA = (32x32 output tile, sample). The tile maps to a rectangle of the flipped, rotated image G (flip and blur commute:
// the Gaussian is symmetric and reflect-101 is mirror-symmetric). Each thread evaluates G on that rectangle plus the
// 2-pixel blur halo (halo indices reflected into G's frame), composing, per value:
//   G(y, x) = R(y, flip ? rw-1-x : x)                                   horizontal flip
//   R(y, x) = cv2 warpAffine INTER_LINEAR of Z in fixed point (AB_BITS 10, 5-bit bilinear fractions, border = mean)
//   Z(y, x) = cv2 resize INTER_LINEAR of the uint8 source (fp32 horizontal pass, then vertical)
// straight from the source bytes, so nothing at resized or rotated resolution exists anywhere. The staged tile is blurred
// separably in shared memory ([1 4 6 4 1]/16, rows first as cv2's sepFilter2D), then padded, normalised and stored
// fp32 NCHW. Labels compose the three integer index maps per output pixel (pad/crop/flip, warp-nearest, resize-nearest).
// A stage whose flag is off is skipped rather than run at identity. No atomics: every output is written once, by one
// thread, from the sample's own descriptor, so it does not depend on the rest of the batch.
#include "host_common.h"

namespace sb {

constexpr int kAugT = 32;                 // output tile edge
constexpr int kAugS = kAugT + 4;          // staged edge (2-pixel blur halo each side)
constexpr int kAugThreads = 256;

struct AugConst {
  float mean[3];
  float std[3];
  int crop_h, crop_w, ignore_label;
};

__device__ __forceinline__ float3 src_px(const uint8_t* __restrict__ img, int w, int y, int x) {
  const uint8_t* p = img + (static_cast<long long>(y) * w + x) * 3;
  return make_float3(static_cast<float>(p[0]), static_cast<float>(p[1]), static_cast<float>(p[2]));
}

// cv2 resize INTER_LINEAR source index and fraction along one axis: s = (d + 0.5) * scale - 0.5 in double, i = floor(s),
// fraction (float)(s - i), clamped at both edges with a zero fraction. A float coordinate (s rounded to fp32 before the
// floor) is off by up to an fp32 ulp of s, which at 2048 columns moves the result by 1e-2 grey levels.
__device__ __forceinline__ void lin_coord(int d, double scale, int n, int& i0, int& i1, float& a) {
  const double s = __dsub_rn(__dmul_rn(static_cast<double>(d) + 0.5, scale), 0.5);
  const double fl = floor(s);
  int i = static_cast<int>(fl);
  float fr = static_cast<float>(__dsub_rn(s, fl));
  if (i < 0) { i = 0; fr = 0.f; }
  if (i >= n - 1) { i = n - 1; fr = 0.f; }
  i0 = i;
  i1 = min(i + 1, n - 1);
  a = fr;
}

// Z(y, x): the resized image (or the source itself under cv2's copy shortcut).
__device__ __forceinline__ float3 resized_px(const semseg_augment_desc& d, const uint8_t* __restrict__ img, int y, int x) {
  if (d.rh == d.h && d.rw == d.w) return src_px(img, d.w, y, x);
  int x0, x1, y0, y1;
  float ax, ay;
  lin_coord(x, d.scale_x, d.w, x0, x1, ax);
  lin_coord(y, d.scale_y, d.h, y0, y1, ay);
  const float bx = 1.f - ax, by = 1.f - ay;
  const float3 p00 = src_px(img, d.w, y0, x0), p01 = src_px(img, d.w, y0, x1);
  const float3 p10 = src_px(img, d.w, y1, x0), p11 = src_px(img, d.w, y1, x1);
  const float3 r0 = make_float3(p00.x * bx + p01.x * ax, p00.y * bx + p01.y * ax, p00.z * bx + p01.z * ax);
  const float3 r1 = make_float3(p10.x * bx + p11.x * ax, p10.y * bx + p11.y * ax, p10.z * bx + p11.z * ax);
  return make_float3(r0.x * by + r1.x * ay, r0.y * by + r1.y * ay, r0.z * by + r1.z * ay);
}

// cv2 warpAffine's fixed-point source position of destination (y, x) (imgproc/imgwarp.cpp, AB_BITS = 10):
// X = rint(M00 x 1024) + rint((M01 y + M02) 1024) + round_delta, and the same for Y.
__device__ __forceinline__ void warp_fixed(const semseg_augment_desc& d, int y, int x, int round_delta, int& X, int& Y) {
  const double xd = static_cast<double>(x), yd = static_cast<double>(y);
  const int adelta = __double2int_rn(__dmul_rn(__dmul_rn(d.m[0], xd), 1024.0));
  const int bdelta = __double2int_rn(__dmul_rn(__dmul_rn(d.m[3], xd), 1024.0));
  const int X0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(d.m[1], yd), d.m[2]), 1024.0)) + round_delta;
  const int Y0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(d.m[4], yd), d.m[5]), 1024.0)) + round_delta;
  X = X0 + adelta;
  Y = Y0 + bdelta;
}

// R(y, x): the rotated image (INTER_LINEAR, 1/32-pixel bilinear weights, constant border = mean).
__device__ __forceinline__ float3 rotated_px(const semseg_augment_desc& d, const uint8_t* __restrict__ img, int y, int x,
                                             const AugConst& k) {
  if (!d.rotate) return resized_px(d, img, y, x);
  int X, Y;
  warp_fixed(d, y, x, 16, X, Y);
  X >>= 5;
  Y >>= 5;
  const int sx = X >> 5, sy = Y >> 5;
  const float tx = static_cast<float>(X & 31) * (1.f / 32.f), ty = static_cast<float>(Y & 31) * (1.f / 32.f);
  const float3 cval = make_float3(k.mean[0], k.mean[1], k.mean[2]);
  if (sx >= d.rw || sx + 1 < 0 || sy >= d.rh || sy + 1 < 0) return cval;
  const float vx0 = 1.f - tx, vy0 = 1.f - ty;
  const float w00 = vy0 * vx0, w01 = vy0 * tx, w10 = ty * vx0, w11 = ty * tx;
  const bool in_x0 = sx >= 0, in_x1 = sx + 1 < d.rw, in_y0 = sy >= 0, in_y1 = sy + 1 < d.rh;
  const float3 p00 = (in_y0 && in_x0) ? resized_px(d, img, sy, sx) : cval;
  const float3 p01 = (in_y0 && in_x1) ? resized_px(d, img, sy, sx + 1) : cval;
  const float3 p10 = (in_y1 && in_x0) ? resized_px(d, img, sy + 1, sx) : cval;
  const float3 p11 = (in_y1 && in_x1) ? resized_px(d, img, sy + 1, sx + 1) : cval;
  return make_float3(p00.x * w00 + p01.x * w01 + p10.x * w10 + p11.x * w11,
                     p00.y * w00 + p01.y * w01 + p10.y * w10 + p11.y * w11,
                     p00.z * w00 + p01.z * w01 + p10.z * w10 + p11.z * w11);
}

// cv2::borderInterpolate(p, n, BORDER_REFLECT_101).
__device__ __forceinline__ int reflect101(int p, int n) {
  if (n == 1) return 0;
  while (p < 0 || p >= n) p = p < 0 ? -p : 2 * n - 2 - p;
  return p;
}

// Label of one output pixel: ignore in the padding and outside the warp, else the composed nearest-neighbour indices.
__device__ __forceinline__ int label_at(const semseg_augment_desc& d, const uint8_t* __restrict__ lab, int gy, int gx,
                                        int ignore) {
  if (gy < 0 || gy >= d.rh || gx < 0 || gx >= d.rw) return ignore;
  int y = gy, x = d.flip ? d.rw - 1 - gx : gx;
  if (d.rotate) {
    int X, Y;
    warp_fixed(d, y, x, 512, X, Y);
    X >>= 10;
    Y >>= 10;
    if (X < 0 || X >= d.rw || Y < 0 || Y >= d.rh) return ignore;
    x = X;
    y = Y;
  }
  if (!(d.rh == d.h && d.rw == d.w)) {     // cv2 resizeNN: min(floor(d * (1/f)), n - 1) in double
    x = min(static_cast<int>(floor(__dmul_rn(static_cast<double>(x), d.scale_x))), d.w - 1);
    y = min(static_cast<int>(floor(__dmul_rn(static_cast<double>(y), d.scale_y))), d.h - 1);
  }
  return lab[static_cast<long long>(y) * d.w + x];
}

__global__ void __launch_bounds__(kAugThreads)
augment_kernel(const uint8_t* __restrict__ data, const semseg_augment_desc* __restrict__ descs, const AugConst k,
               float* __restrict__ out_img, long long* __restrict__ out_lab) {
  __shared__ float s_g[3][kAugS][kAugS + 1];       // G on the tile + halo
  __shared__ float s_h[3][kAugS][kAugT + 1];       // after the horizontal blur pass
  const int n = blockIdx.z;
  const semseg_augment_desc d = descs[n];
  const uint8_t* __restrict__ img = data + d.img_off;
  const uint8_t* __restrict__ lab = data + d.lab_off;
  const int oy0 = blockIdx.y * kAugT, ox0 = blockIdx.x * kAugT;
  // G-frame coordinate of the tile's first output pixel
  const int gy0 = oy0 + d.off_y - d.pad_top, gx0 = ox0 + d.off_x - d.pad_left;
  const bool any = gy0 + kAugT > 0 && gy0 < d.rh && gx0 + kAugT > 0 && gx0 < d.rw;
  const int tid = threadIdx.x;

  if (any) {
    const int lo = d.blur ? 0 : 2, hi = d.blur ? kAugS : kAugS - 2;
    const int span = hi - lo;
    for (int i = tid; i < span * span; i += kAugThreads) {
      const int sy = lo + i / span, sx = lo + i % span;
      int gy = gy0 - 2 + sy, gx = gx0 - 2 + sx;
      float3 v = make_float3(0.f, 0.f, 0.f);
      // only values within 2 pixels of G's frame are read by an in-frame output pixel
      if (gy >= -2 && gy < d.rh + 2 && gx >= -2 && gx < d.rw + 2) {
        gy = reflect101(gy, d.rh);
        gx = reflect101(gx, d.rw);
        v = rotated_px(d, img, gy, d.flip ? d.rw - 1 - gx : gx, k);
      }
      s_g[0][sy][sx] = v.x;
      s_g[1][sy][sx] = v.y;
      s_g[2][sy][sx] = v.z;
    }
    __syncthreads();
    if (d.blur) {
      for (int i = tid; i < 3 * kAugS * kAugT; i += kAugThreads) {
        const int c = i / (kAugS * kAugT), r = (i / kAugT) % kAugS, x = i % kAugT;
        const float* row = &s_g[c][r][x];
        s_h[c][r][x] = row[0] * 0.0625f + row[1] * 0.25f + row[2] * 0.375f + row[3] * 0.25f + row[4] * 0.0625f;
      }
      __syncthreads();
    }
  }

  const long long plane = static_cast<long long>(k.crop_h) * k.crop_w;
  for (int i = tid; i < kAugT * kAugT; i += kAugThreads) {
    const int ty = i / kAugT, tx = i % kAugT;
    const int oy = oy0 + ty, ox = ox0 + tx;
    if (oy >= k.crop_h || ox >= k.crop_w) continue;
    const int gy = gy0 + ty, gx = gx0 + tx;
    const bool inside = gy >= 0 && gy < d.rh && gx >= 0 && gx < d.rw;
    const long long o = static_cast<long long>(oy) * k.crop_w + ox;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float v = 0.f;
      if (inside) {
        float g;
        if (d.blur) {
          g = s_h[c][ty][tx] * 0.0625f + s_h[c][ty + 1][tx] * 0.25f + s_h[c][ty + 2][tx] * 0.375f +
              s_h[c][ty + 3][tx] * 0.25f + s_h[c][ty + 4][tx] * 0.0625f;
        } else {
          g = s_g[c][ty + 2][tx + 2];
        }
        v = (g - k.mean[c]) / k.std[c];
      }
      out_img[(static_cast<long long>(n) * 3 + c) * plane + o] = v;     // padding: (mean - mean) / std = 0
    }
    out_lab[static_cast<long long>(n) * plane + o] = label_at(d, lab, gy, gx, k.ignore_label);
  }
}

}  // namespace sb

extern "C" int semseg_augment(const void* data, long long data_bytes, const semseg_augment_desc* desc_host,
                              const semseg_augment_desc* desc_dev, int n, int crop_h, int crop_w, const float* mean3,
                              const float* std3, int ignore_label, float* out_img, long long* out_lab, void* stream_) {
  SB_CHECK_ARG(data && desc_host && desc_dev && mean3 && std3 && out_img && out_lab, "augment: null pointer");
  SB_CHECK_ARG(n > 0 && n <= 65535, "augment: batch of %d samples (1..65535)", n);
  SB_CHECK_ARG(crop_h > 0 && crop_w > 0, "augment: crop %dx%d must be positive", crop_h, crop_w);
  SB_CHECK_ARG(data_bytes > 0, "augment: empty data buffer");
  for (int c = 0; c < 3; ++c) SB_CHECK_ARG(std3[c] != 0.f, "augment: std[%d] is zero", c);
  for (int i = 0; i < n; ++i) {
    const semseg_augment_desc& d = desc_host[i];
    SB_CHECK_ARG(d.h > 0 && d.w > 0 && d.rh > 0 && d.rw > 0, "augment: sample %d has size %dx%d -> %dx%d", i, d.h, d.w,
                 d.rh, d.rw);
    SB_CHECK_ARG(d.img_off >= 0 && d.img_off + 3LL * d.h * d.w <= data_bytes,
                 "augment: sample %d image [%lld, +%lld) outside the %lld-byte buffer", i, d.img_off, 3LL * d.h * d.w,
                 data_bytes);
    SB_CHECK_ARG(d.lab_off >= 0 && d.lab_off + 1LL * d.h * d.w <= data_bytes,
                 "augment: sample %d label [%lld, +%lld) outside the %lld-byte buffer", i, d.lab_off, 1LL * d.h * d.w,
                 data_bytes);
    const bool resize = !(d.rh == d.h && d.rw == d.w);
    SB_CHECK_ARG(!resize || (d.scale_x > 0.0 && d.scale_y > 0.0), "augment: sample %d resize step must be positive", i);
    SB_CHECK_ARG((d.rotate == 0 || d.rotate == 1) && (d.blur == 0 || d.blur == 1) && (d.flip == 0 || d.flip == 1),
                 "augment: sample %d flags must be 0 or 1", i);
    const int ph = crop_h > d.rh ? crop_h - d.rh : 0, pw = crop_w > d.rw ? crop_w - d.rw : 0;
    SB_CHECK_ARG(d.pad_top == ph / 2 && d.pad_left == pw / 2, "augment: sample %d padding (%d, %d) != (%d, %d)", i,
                 d.pad_top, d.pad_left, ph / 2, pw / 2);
    SB_CHECK_ARG(d.off_y >= 0 && d.off_y <= d.rh + ph - crop_h && d.off_x >= 0 && d.off_x <= d.rw + pw - crop_w,
                 "augment: sample %d crop offset (%d, %d) outside the padded %dx%d image", i, d.off_y, d.off_x,
                 d.rh + ph, d.rw + pw);
  }
  sb::AugConst k;
  for (int c = 0; c < 3; ++c) {
    k.mean[c] = mean3[c];
    k.std[c] = std3[c];
  }
  k.crop_h = crop_h;
  k.crop_w = crop_w;
  k.ignore_label = ignore_label;
  const dim3 grid(static_cast<unsigned>(sb::cdiv(crop_w, sb::kAugT)), static_cast<unsigned>(sb::cdiv(crop_h, sb::kAugT)),
                  static_cast<unsigned>(n));
  SB_CHECK_ARG(grid.y <= 65535, "augment: crop height %d too large", crop_h);
  sb::augment_kernel<<<grid, sb::kAugThreads, 0, static_cast<cudaStream_t>(stream_)>>>(
      static_cast<const uint8_t*>(data), desc_dev, k, out_img, out_lab);
  SB_LAUNCHED();
  return SEMSEG_OK;
}
