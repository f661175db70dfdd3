// HBM-bound helper kernels around the conv path: boundary layout adapters, stem space-to-depth,
// SPPF pooling and the YOLOv5 per-anchor decode.  All are plain coalesced/vectorised CUDA; none is GEMM shaped.
#include <cuda_fp16.h>
#include <math_constants.h>

#include "internal.h"

namespace cvb {

// ------------------------------------------------------------------ NCHW fp32 -> split16 NHWC
// grid (ceil(W/32), ceil(C/32), image rows), block (32, 8): smem transpose so both sides are coalesced.  Image row b*H + h =
// bh0 + blockIdx.z: the host launches chunks of at most kMaxGridZ rows (the grid's z limit), so any B*H converts.
constexpr int kMaxGridZ = 65535;

__global__ void nchw_to_split_kernel(const float* __restrict__ src, int B, int C, int H, int W, __half* __restrict__ dst, int pitch,
                                     long long plane, int bh0) {
  __shared__ float tile[32][33];
  const int bh = bh0 + (int)blockIdx.z;
  const int b = bh / H, h = bh % H;
  const int w0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int c = c0 + i, w = w0 + threadIdx.x;
    tile[i][threadIdx.x] = (c < C && w < W) ? src[(((size_t)b * C + c) * H + h) * W + w] : 0.0f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int w = w0 + i, c = c0 + threadIdx.x;
    if (w < W && c < C) {
      const float v = tile[threadIdx.x][i];
      uint32_t hi, lo;
      split_pair(v, v, hi, lo);
      const size_t o = (((size_t)b * H + h) * W + w) * pitch + c;
      dst[o] = __ushort_as_half((unsigned short)hi);
      dst[o + plane] = __ushort_as_half((unsigned short)lo);
    }
  }
}

// split16 NHWC -> NCHW fp32 (x = hi + lo)
__global__ void split_to_nchw_kernel(const __half* __restrict__ src, int B, int C, int H, int W, int pitch, long long plane,
                                     float* __restrict__ dst, int bh0) {
  __shared__ float tile[32][33];
  const int bh = bh0 + (int)blockIdx.z;
  const int b = bh / H, h = bh % H;
  const int w0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int w = w0 + i, c = c0 + threadIdx.x;
    float v = 0.0f;
    if (w < W && c < C) {
      const size_t o = (((size_t)b * H + h) * W + w) * pitch + c;
      v = __half2float(src[o]) + __half2float(src[o + plane]);
    }
    tile[i][threadIdx.x] = v;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int c = c0 + i, w = w0 + threadIdx.x;
    if (c < C && w < W) dst[(((size_t)b * C + c) * H + h) * W + w] = tile[threadIdx.x][i];
  }
}

__global__ void f32nhwc_to_nchw_kernel(const float* __restrict__ src, int B, int C, int H, int W, int pitch, float* __restrict__ dst,
                                       int bh0) {
  __shared__ float tile[32][33];
  const int bh = bh0 + (int)blockIdx.z;
  const int b = bh / H, h = bh % H;
  const int w0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int w = w0 + i, c = c0 + threadIdx.x;
    tile[i][threadIdx.x] = (w < W && c < C) ? src[(((size_t)b * H + h) * W + w) * pitch + c] : 0.0f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int c = c0 + i, w = w0 + threadIdx.x;
    if (c < C && w < W) dst[(((size_t)b * C + c) * H + h) * W + w] = tile[threadIdx.x][i];
  }
}

// ------------------------------------------------------------------ stem space-to-depth
// One thread per output pixel (b, h2, w2): reads a 2x2x3 patch (float2 per row/channel -> coalesced across
// the warp) and writes 16 channels (12 used) as two 32-byte hi/lo records (coalesced across the warp).
__global__ void stem_s2d_kernel(const float* __restrict__ src, int B, int H, int W, __half* __restrict__ dst, int pitch,
                                long long plane, int Wd, int col_off) {
  const int W2 = W >> 1, H2 = H >> 1;
  const long long n = (long long)B * H2 * W2;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int w2 = (int)(i % W2);
    const long long t = i / W2;
    const int h2 = (int)(t % H2);
    const int b = (int)(t / H2);
    float v[16];
#pragma unroll
    for (int k = 12; k < 16; ++k) v[k] = 0.0f;
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
      for (int dy = 0; dy < 2; ++dy) {
        const float2 p = __ldg(reinterpret_cast<const float2*>(src + (((size_t)b * 3 + c) * H + (2 * h2 + dy)) * W + 2 * w2));
        v[(dy * 2 + 0) * 3 + c] = p.x;
        v[(dy * 2 + 1) * 3 + c] = p.y;
      }
    uint32_t hq[8], lq[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      split_pair(v[2 * k], v[2 * k + 1], hq[k], lq[k]);
    }
    __half* o = dst + (((size_t)b * H2 + h2) * Wd + (w2 + col_off)) * pitch;  // Wd > W2: zero-padded row-window layout
    reinterpret_cast<uint4*>(o)[0] = make_uint4(hq[0], hq[1], hq[2], hq[3]);
    reinterpret_cast<uint4*>(o)[1] = make_uint4(hq[4], hq[5], hq[6], hq[7]);
    reinterpret_cast<uint4*>(o + plane)[0] = make_uint4(lq[0], lq[1], lq[2], lq[3]);
    reinterpret_cast<uint4*>(o + plane)[1] = make_uint4(lq[4], lq[5], lq[6], lq[7]);
  }
}

// Same output, fed by the camera-side format: uint8 HWC frames.  ToTensor (src/data/transforms/det_transforms.py:85-99: HWC->CHW,
// channel reversal BGR->RGB, float32 / 255) and Normalize (:102-109, torchvision F.normalize: (x - mean) / std in fp32) are
// applied while the 2x2x3 patch is in registers, with the reference's operation order and IEEE division, so the result is
// bit-identical to stem_s2d_kernel on the tensor the reference's transforms would have produced.  One thread per output pixel:
// reads 2 rows x 6 contiguous bytes.
// A 256-entry table per output channel (built per CTA with exactly those operations) replaces 24 IEEE divisions per thread.
// PAIR: one thread converts two horizontally adjacent output pixels = 12 contiguous source bytes per row (three aligned 32-bit
// loads; needs W % 4 == 0); otherwise one output pixel per thread with 16-bit loads.
template <bool PAIR>
__global__ void __launch_bounds__(256) stem_s2d_u8_kernel(const uint8_t* __restrict__ src, int B, int H, int W, float m0, float m1, float m2,
                                                          float s0, float s1, float s2, int reverse, __half* __restrict__ dst, int pitch,
                                                          long long plane, int Wd, int col_off) {
  __shared__ float lut[3][256];  // lut[c][byte] for OUTPUT channel c
  {
    const float mean[3] = {m0, m1, m2}, stdv[3] = {s0, s1, s2};
    for (int i = threadIdx.x; i < 768; i += blockDim.x) {
      const int c = i >> 8;
      lut[c][i & 255] = __fdiv_rn(__fsub_rn(__fdiv_rn((float)(i & 255), 255.0f), mean[c]), stdv[c]);
    }
  }
  __syncthreads();
  const int W2 = W >> 1, H2 = H >> 1;
  constexpr int PX = PAIR ? 2 : 1;
  const int Wt = W2 / PX;
  const long long n = (long long)B * H2 * Wt;
  const int cmap0 = reverse ? 2 : 0, cmap2 = reverse ? 0 : 2;  // output channel of source channels 0 and 2 (1 stays 1)
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int wt = (int)(i % Wt);
    const long long t = i / Wt;
    const int h2 = (int)(t % H2);
    const int b = (int)(t / H2);
    const int w2 = wt * PX;
    uint8_t px[2][6 * PX];
#pragma unroll
    for (int dy = 0; dy < 2; ++dy) {
      const uint8_t* p = src + (((size_t)b * H + (2 * h2 + dy)) * W + 2 * w2) * 3;
      if constexpr (PAIR) {
        const uint32_t* p4 = reinterpret_cast<const uint32_t*>(p);
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const uint32_t a = __ldg(p4 + k);
          px[dy][4 * k + 0] = (uint8_t)(a & 0xFF);
          px[dy][4 * k + 1] = (uint8_t)((a >> 8) & 0xFF);
          px[dy][4 * k + 2] = (uint8_t)((a >> 16) & 0xFF);
          px[dy][4 * k + 3] = (uint8_t)(a >> 24);
        }
      } else {
        const uint16_t* p2 = reinterpret_cast<const uint16_t*>(p);
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const uint32_t a = __ldg(p2 + k);
          px[dy][2 * k + 0] = (uint8_t)(a & 0xFF);
          px[dy][2 * k + 1] = (uint8_t)(a >> 8);
        }
      }
    }
#pragma unroll
    for (int q = 0; q < PX; ++q) {
      float v[16];
#pragma unroll
      for (int k = 12; k < 16; ++k) v[k] = 0.0f;
#pragma unroll
      for (int dy = 0; dy < 2; ++dy)
#pragma unroll
        for (int dx = 0; dx < 2; ++dx) {
          const uint8_t* s3 = &px[dy][(q * 2 + dx) * 3];
          v[(dy * 2 + dx) * 3 + cmap0] = lut[cmap0][s3[0]];
          v[(dy * 2 + dx) * 3 + 1] = lut[1][s3[1]];
          v[(dy * 2 + dx) * 3 + cmap2] = lut[cmap2][s3[2]];
        }
      uint32_t hq[8], lq[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        split_pair(v[2 * k], v[2 * k + 1], hq[k], lq[k]);
      }
      __half* o = dst + (((size_t)b * H2 + h2) * Wd + (w2 + q + col_off)) * pitch;
      reinterpret_cast<uint4*>(o)[0] = make_uint4(hq[0], hq[1], hq[2], hq[3]);
      reinterpret_cast<uint4*>(o)[1] = make_uint4(hq[4], hq[5], hq[6], hq[7]);
      reinterpret_cast<uint4*>(o + plane)[0] = make_uint4(lq[0], lq[1], lq[2], lq[3]);
      reinterpret_cast<uint4*>(o + plane)[1] = make_uint4(lq[4], lq[5], lq[6], lq[7]);
    }
  }
}

// ------------------------------------------------------------------ SPPF: three chained 5x5/s1/p2 max pools
// One CTA per (image, 8-channel slice): the whole HxW map of the slice lives in shared memory as fp32;
// each pool is a separable row-max / column-max pass.  y2 == 9x9 pool, y3 == 13x13 pool of x.  NaN propagates (nan_max).
__global__ void sppf_pool_kernel(const __half* __restrict__ x, int H, int W, int xp, long long xplane, __half* __restrict__ y1, int p1,
                                 long long plane1, __half* __restrict__ y2, int p2, long long plane2, __half* __restrict__ y3, int p3,
                                 long long plane3, int cgroups) {
  extern __shared__ float sm[];
  float* cur = sm;                 // [H*W][8]
  float* tmp = sm + (size_t)H * W * 8;
  const int b = blockIdx.x / cgroups;
  const int c0 = (blockIdx.x % cgroups) * 8;
  const int npix = H * W;
  for (int p = threadIdx.x; p < npix; p += blockDim.x) {
    const size_t o = ((size_t)b * npix + p) * xp + c0;
    const uint4 hv = *reinterpret_cast<const uint4*>(x + o);
    const uint4 lv = *reinterpret_cast<const uint4*>(x + o + xplane);
    const __half2* h2 = reinterpret_cast<const __half2*>(&hv);
    const __half2* l2 = reinterpret_cast<const __half2*>(&lv);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      cur[p * 8 + 2 * k] = __low2float(h2[k]) + __low2float(l2[k]);
      cur[p * 8 + 2 * k + 1] = __high2float(h2[k]) + __high2float(l2[k]);
    }
  }
  __syncthreads();
  __half* outs[3] = {y1, y2, y3};
  const int pitches[3] = {p1, p2, p3};
  const long long planes[3] = {plane1, plane2, plane3};
  for (int r = 0; r < 3; ++r) {
    // row pass: tmp[h][w] = max_{|d|<=2} cur[h][w+d]; one thread per (pixel, 4-channel vector)
    const float4* cur4 = reinterpret_cast<const float4*>(cur);
    float4* tmp4 = reinterpret_cast<float4*>(tmp);
    for (int i = threadIdx.x; i < npix * 2; i += blockDim.x) {
      const int hf = i & 1, p = i >> 1, h = p / W, w = p - h * W;
      float4 m = cur4[i];
#pragma unroll
      for (int d = -2; d <= 2; ++d) {
        const int ww = w + d;
        if (d != 0 && ww >= 0 && ww < W) {
          const float4 v = cur4[(p + d) * 2 + hf];
          m.x = nan_max(m.x, v.x);
          m.y = nan_max(m.y, v.y);
          m.z = nan_max(m.z, v.z);
          m.w = nan_max(m.w, v.w);
        }
      }
      tmp4[i] = m;
    }
    __syncthreads();
    float4* curw4 = reinterpret_cast<float4*>(cur);
    for (int i = threadIdx.x; i < npix * 2; i += blockDim.x) {
      const int hf = i & 1, p = i >> 1, h = p / W;
      float4 m = tmp4[i];
#pragma unroll
      for (int d = -2; d <= 2; ++d) {
        const int hh = h + d;
        if (d != 0 && hh >= 0 && hh < H) {
          const float4 v = tmp4[(p + d * W) * 2 + hf];
          m.x = nan_max(m.x, v.x);
          m.y = nan_max(m.y, v.y);
          m.z = nan_max(m.z, v.z);
          m.w = nan_max(m.w, v.w);
        }
      }
      curw4[i] = m;
    }
    __syncthreads();
    for (int p = threadIdx.x; p < npix; p += blockDim.x) {
      uint32_t hq[4], lq[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        split_pair(cur[p * 8 + 2 * k], cur[p * 8 + 2 * k + 1], hq[k], lq[k]);
      }
      const size_t o = ((size_t)b * npix + p) * pitches[r] + c0;
      *reinterpret_cast<uint4*>(outs[r] + o) = make_uint4(hq[0], hq[1], hq[2], hq[3]);
      *reinterpret_cast<uint4*>(outs[r] + o + planes[r]) = make_uint4(lq[0], lq[1], lq[2], lq[3]);
    }
    // cur stays as the input of the next chained pool
  }
}

// ------------------------------------------------------------------ YOLOv5 decode
// Grid (pixel chunks, B); one warp per output row (anchor a, pixel), anchor-major: three 32-lane chunks of the row's no <= 96 floats
// are read and written coalesced, kDecodeRows rows in flight.  While the scores are in registers the CTA also builds the NMS score
// histogram of its image in shared memory (64 KB, HIST) and flushes the non-empty bins once -- this replaces the separate counting
// pass over the 548 MB prediction tensor and keeps the hot bins out of global atomics.  MULTI: one histogram entry per class score
// above conf, else one per row (its best score).  z may be null without HIST; xperm (the raw rows, permuted) may be null.
constexpr int kDecodePix = 512;      // pixels per CTA (x na anchor rows)
constexpr int kDecodeThreads = 512;  // 16 warps
constexpr int kDecodeRows = 4;       // rows in flight per warp (all loads issued before the first use)

template <bool HIST, bool MULTI>
__global__ void __launch_bounds__(kDecodeThreads) yolo_decode_kernel(const float* __restrict__ raw, int ny, int nx, int pitch, int na,
                                                                     int no, const float* __restrict__ anchors_px, float stride,
                                                                     float* __restrict__ z, long long z_rows, long long z_off,
                                                                     float* __restrict__ xperm, uint32_t* __restrict__ hist,
                                                                     float* __restrict__ rowmax, float conf, uint32_t nx_magic) {
  extern __shared__ uint32_t s_hist[];  // [kNmsBins] when HIST
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr int NW = kDecodeThreads / 32;
  constexpr int R = kDecodeRows;
  const int b = blockIdx.y;
  const int npix = ny * nx;
  const int pix0 = blockIdx.x * kDecodePix;
  const int cpix = min(npix, pix0 + kDecodePix) - pix0;
  if (HIST) nms_hist_clear<kDecodeThreads>(s_hist);
  const float* rbase = raw + ((size_t)b * npix + pix0) * pitch;
  const size_t zb = ((size_t)b * z_rows + z_off) * no;  // z element of the level's first row in image b
  const size_t xb = (size_t)b * na * npix * no;
  float* rmb = HIST ? rowmax + (size_t)b * z_rows + z_off : nullptr;
  const bool v0 = lane < no, v1 = 32 + lane < no, v2 = 64 + lane < no;
  const bool is_cls = v0 && lane >= 5;
  for (int a = 0; a < na; ++a) {
    const float anchor = __ldg(anchors_px + a * 2 + (lane & 1));  // w (even lanes) or h (odd lanes) of this anchor, in pixels
    for (int p0 = warp * R; p0 < cpix; p0 += NW * R) {
      float v[R][3];
#pragma unroll
      for (int i = 0; i < R; ++i) {
        const int p = min(p0 + i, cpix - 1);
        const float* src = rbase + (size_t)(uint32_t)p * (uint32_t)pitch + (uint32_t)(a * no + lane);
        v[i][0] = v0 ? __ldg(src) : 0.0f;
        v[i][1] = v1 ? __ldg(src + 32) : 0.0f;
        v[i][2] = v2 ? __ldg(src + 64) : 0.0f;
      }
      int pyv[R];  // pixel row of every row in flight, computed before the row loop (keeps fast_div's branches out of it)
#pragma unroll
      for (int i = 0; i < R; ++i) pyv[i] = fast_div(pix0 + min(p0 + i, cpix - 1), nx, nx_magic);
      if (xperm != nullptr) {  // kernel-uniform: copy the raw rows
#pragma unroll
        for (int i = 0; i < R; ++i) {
          if (p0 + i < cpix) {
            float* dst = xperm + xb + (size_t)(uint32_t)(a * npix + pix0 + p0 + i) * no + lane;
            if (v0) dst[0] = v[i][0];
            if (v1) dst[32] = v[i][1];
            if (v2) dst[64] = v[i][2];
          }
        }
      }
#pragma unroll
      for (int i = 0; i < R; ++i) {
        const bool ok = (p0 + i) < cpix;  // tail rows are computed on clamped inputs and not stored (keeps the shuffles convergent)
        const int pix = pix0 + min(p0 + i, cpix - 1);
        // this lane's element of level row a * npix + pix (na * npix < 2^31: checked on the host)
        const size_t roff = (size_t)(uint32_t)(a * npix + pix) * no + lane;
        const int py = pyv[i], px = pix - py * nx;
        const float y0 = sigmoid_fast(v[i][0]);
        const float y1 = sigmoid_fast(v[i][1]);
        const float y2 = sigmoid_fast(v[i][2]);
        const float xy = yolo_xy(y0, lane == 0 ? (float)px : (float)py, stride);
        const float wh = yolo_wh(y0, anchor);
        const float o0 = lane < 2 ? xy : (lane < 4 ? wh : y0);
        if (ok && z != nullptr) {
          float* dst = z + zb + roff;
          if (v0) dst[0] = o0;
          if (v1) dst[32] = y1;
          if (v2) dst[64] = y2;
        }
        if (HIST) {
          const float obj = __shfl_sync(0xffffffffu, o0, 4);
          float rbest = 0.0f;
          if (ok && obj > conf) {  // warp-uniform
            nms_count_score(s_hist, is_cls ? yolo_score(o0, obj) : 0.0f, conf, MULTI, rbest);
            nms_count_score(s_hist, v1 ? yolo_score(y1, obj) : 0.0f, conf, MULTI, rbest);
            nms_count_score(s_hist, v2 ? yolo_score(y2, obj) : 0.0f, conf, MULTI, rbest);
            rbest = nms_finish_row(s_hist, rbest, conf, MULTI, lane);
          }
          if (ok && lane == 0) rmb[a * npix + pix] = rbest;
        }
      }
    }
  }
  if (HIST) nms_hist_flush<kDecodeThreads>(s_hist, hist + (size_t)b * kNmsBins);
}

// ------------------------------------------------------------------ YOLOv6 anchor-free decode
// Grid (pixel chunks, B); one warp per z row (one anchor per pixel), its no = 5 + nc <= 96 floats in three coalesced 32-lane chunks:
// lanes 0..3 the box, lane 4 the objectness 1.0, the rest sigmoid(class logit).  Box: anchor (x + 0.5, y + 0.5), x1y1 = a - lt,
// x2y2 = a + rb, centre (x1y1 + x2y2) / 2, size x2y2 - x1y1, times stride -- dist2bbox(..., 'xywh') of yolov6_loss.py:205-216 in its
// fp32 operation order.  HIST / MULTI: the NMS pre-pass of yolo_decode_kernel with obj = 1, so score = cls * 1 = cls bit for bit.
constexpr int kV6DecodePix = 256;  // pixels per CTA
constexpr int kV6DecodeThreads = 256;

template <bool HIST, bool MULTI>
__global__ void __launch_bounds__(kV6DecodeThreads) yolov6_decode_kernel(const float* __restrict__ cls, int cls_pitch, const float* __restrict__ reg,
                                                                         int reg_pitch, int ny, int nx, int nc, float stride,
                                                                         float* __restrict__ z, long long z_rows, long long z_off,
                                                                         uint32_t* __restrict__ hist, float* __restrict__ rowmax, float conf) {
  extern __shared__ uint32_t s_hist[];  // [kNmsBins] when HIST
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr int NW = kV6DecodeThreads / 32;
  const int b = blockIdx.y;
  const int npix = ny * nx;
  const int pix0 = blockIdx.x * kV6DecodePix;
  const int cpix = min(npix, pix0 + kV6DecodePix) - pix0;
  const int no = nc + 5;
  if (HIST) nms_hist_clear<kV6DecodeThreads>(s_hist);
  const bool v0 = lane < no, v1 = 32 + lane < no, v2 = 64 + lane < no;
  const bool is_cls = v0 && lane >= 5;
  float* rmb = HIST ? rowmax + (size_t)b * z_rows + z_off : nullptr;
  for (int p = warp; p < cpix; p += NW) {  // warp-uniform loop
    const int pix = pix0 + p;
    const size_t q = (size_t)b * npix + pix;
    const float* cr = cls + q * cls_pitch;
    const float c0 = is_cls ? __ldg(cr + lane - 5) : 0.0f;
    const float c1 = v1 ? __ldg(cr + lane + 27) : 0.0f;
    const float c2 = v2 ? __ldg(cr + lane + 59) : 0.0f;
    float o0;
    if (lane < 4) {
      const int d = lane & 1;  // 0: x, 1: y
      const float lt = __ldg(reg + q * reg_pitch + d), rb = __ldg(reg + q * reg_pitch + d + 2);
      const int py = pix / nx;
      const float a = __fadd_rn((float)(d ? py : pix - py * nx), 0.5f);
      const float x1 = __fsub_rn(a, lt), x2 = __fadd_rn(a, rb);
      o0 = __fmul_rn(lane < 2 ? __fmul_rn(__fadd_rn(x1, x2), 0.5f) : __fsub_rn(x2, x1), stride);
    } else {
      o0 = lane == 4 ? 1.0f : sigmoid_fast(c0);
    }
    const float y1 = sigmoid_fast(c1), y2 = sigmoid_fast(c2);
    float* dst = z + ((size_t)b * z_rows + z_off + pix) * no + lane;
    if (v0) dst[0] = o0;
    if (v1) dst[32] = y1;
    if (v2) dst[64] = y2;
    if (HIST) {
      const float obj = 1.0f;  // > conf for every conf_thres < 1 (the NMS refuses larger ones)
      float rbest = 0.0f;
      nms_count_score(s_hist, is_cls ? yolo_score(o0, obj) : 0.0f, conf, MULTI, rbest);
      nms_count_score(s_hist, v1 ? yolo_score(y1, obj) : 0.0f, conf, MULTI, rbest);
      nms_count_score(s_hist, v2 ? yolo_score(y2, obj) : 0.0f, conf, MULTI, rbest);
      rbest = nms_finish_row(s_hist, rbest, conf, MULTI, lane);
      if (lane == 0) rmb[pix] = rbest;
    }
  }
  if (HIST) nms_hist_flush<kV6DecodeThreads>(s_hist, hist + (size_t)b * kNmsBins);
}

// ------------------------------------------------------------------ 2x depth-to-space (ConvTranspose2d k = s = 2 after its 1x1 GEMM)
// src [B,h,w,4c] split16 with channel (py*2+px)*c + o  ->  dst [B,2h,2w,c] split16 pixel (2y+py, 2x+px) channel o.  One thread per (output
// pixel, 8-channel vector); the hi and lo planes are copied as they are, so the values are the GEMM's bit for bit.
__global__ void __launch_bounds__(256) depth_to_space2_kernel(const __half* __restrict__ src, int sp, long long splane, int h, int w, int c,
                                                              __half* __restrict__ dst, int dp, long long dplane, long long n) {
  const int cv = c / 8;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % cv);
    long long r = i / cv;
    const int ox = (int)(r % (2 * w));
    r /= 2 * w;
    const int oy = (int)(r % (2 * h));
    const long long b = r / (2 * h);
    const size_t s = (((size_t)b * h + (oy >> 1)) * w + (ox >> 1)) * sp + (size_t)(((oy & 1) * 2 + (ox & 1)) * c + v * 8);
    const size_t d = (((size_t)b * 2 * h + oy) * 2 * w + ox) * dp + (size_t)v * 8;
    const uint4 hi = *reinterpret_cast<const uint4*>(src + s);
    const uint4 lo = *reinterpret_cast<const uint4*>(src + s + splane);
    *reinterpret_cast<uint4*>(dst + d) = hi;
    *reinterpret_cast<uint4*>(dst + d + dplane) = lo;
  }
}

// ------------------------------------------------------------------ 3x3 / stride 2 / pad 1 max pool (ResNet stem)
// one thread per (output pixel, 8-channel vector); max over hi+lo values, result re-split exactly (max is one of the inputs).  A NaN
// is taken and then kept, like F.max_pool2d; the running maximum starts as -inf (hi = 0xFC00) so an all -inf window gives -inf.
__global__ void maxpool3x3s2_kernel(const __half* __restrict__ x, int B, int H, int W, int C, int xp, long long xplane,
                                    __half* __restrict__ y, int Ho, int Wo, int yp, long long yplane) {
  const int cv = C / 8;
  const long long n = (long long)B * Ho * Wo * cv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(i % cv);
    long long t = i / cv;
    const int wo = (int)(t % Wo);
    t /= Wo;
    const int ho = (int)(t % Ho);
    const int b = (int)(t / Ho);
    float best[8];
    uint4 bh = make_uint4(0xFC00FC00u, 0xFC00FC00u, 0xFC00FC00u, 0xFC00FC00u), bl = make_uint4(0, 0, 0, 0);
    uint32_t* bhw = reinterpret_cast<uint32_t*>(&bh);
    uint32_t* blw = reinterpret_cast<uint32_t*>(&bl);
#pragma unroll
    for (int k = 0; k < 8; ++k) best[k] = -CUDART_INF_F;
    for (int dy = -1; dy <= 1; ++dy) {
      const int h = 2 * ho + dy;
      if (h < 0 || h >= H) continue;
      for (int dx = -1; dx <= 1; ++dx) {
        const int w = 2 * wo + dx;
        if (w < 0 || w >= W) continue;
        const size_t o = (((size_t)b * H + h) * W + w) * xp + c8 * 8;
        const uint4 hv = __ldg(reinterpret_cast<const uint4*>(x + o));
        const uint4 lv = __ldg(reinterpret_cast<const uint4*>(x + o + xplane));
        const uint32_t* hw = reinterpret_cast<const uint32_t*>(&hv);
        const uint32_t* lw = reinterpret_cast<const uint32_t*>(&lv);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hw[e]));
          const float2 lf = __half22float2(*reinterpret_cast<const __half2*>(&lw[e]));
          const float v0 = hf.x + lf.x, v1 = hf.y + lf.y;
          if (v0 > best[2 * e] || (v0 != v0 && best[2 * e] == best[2 * e])) {
            best[2 * e] = v0;
            bhw[e] = (bhw[e] & 0xFFFF0000u) | (hw[e] & 0xFFFFu);
            blw[e] = (blw[e] & 0xFFFF0000u) | (lw[e] & 0xFFFFu);
          }
          if (v1 > best[2 * e + 1] || (v1 != v1 && best[2 * e + 1] == best[2 * e + 1])) {
            best[2 * e + 1] = v1;
            bhw[e] = (bhw[e] & 0xFFFFu) | (hw[e] & 0xFFFF0000u);
            blw[e] = (blw[e] & 0xFFFFu) | (lw[e] & 0xFFFF0000u);
          }
        }
      }
    }
    const size_t oo = (((size_t)b * Ho + ho) * Wo + wo) * yp + c8 * 8;
    *reinterpret_cast<uint4*>(y + oo) = bh;
    *reinterpret_cast<uint4*>(y + oo + yplane) = bl;
  }
}

// ------------------------------------------------------------------ split16 -> fp32 NHWC (FPN partials)
__global__ void split_to_f32_kernel(const __half* __restrict__ x, long long npix, int C, int xp, long long xplane, float* __restrict__ y,
                                    int yp) {
  const int cv = C / 8;
  const long long n = npix * cv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(i % cv);
    const long long p = i / cv;
    const uint4 hv = __ldg(reinterpret_cast<const uint4*>(x + p * xp + c8 * 8));
    const uint4 lv = __ldg(reinterpret_cast<const uint4*>(x + p * xp + c8 * 8 + xplane));
    const uint32_t* hw = reinterpret_cast<const uint32_t*>(&hv);
    const uint32_t* lw = reinterpret_cast<const uint32_t*>(&lv);
    float o[8];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hw[e]));
      const float2 lf = __half22float2(*reinterpret_cast<const __half2*>(&lw[e]));
      o[2 * e] = hf.x + lf.x;
      o[2 * e + 1] = hf.y + lf.y;
    }
    float4* dst = reinterpret_cast<float4*>(y + p * yp + c8 * 8);
    dst[0] = make_float4(o[0], o[1], o[2], o[3]);
    dst[1] = make_float4(o[4], o[5], o[6], o[7]);
  }
}

// ------------------------------------------------------------------ GroupNorm(+ReLU) for 8 channels per group (FCOS towers)
// pivot of (image b, group g): the group's first channel at the image's first pixel.  The sums are taken around it so that they stay at the
// scale of the group's spread: E[x^2] - mean^2 would lose (mean / std)^2 times the fp32 accumulation error.
__device__ __forceinline__ float gn_pivot(const __half* __restrict__ x, int b, int g, int npix, int xp, long long xplane) {
  const size_t o = (size_t)b * npix * xp + g * 8;
  return __half2float(x[o]) + __half2float(x[o + xplane]);
}

// pass 1: per (image, group) sum and sum of squares of x - pivot (fp32 per thread over <= 64 values, double across threads)
__global__ void gn_stats_kernel(const __half* __restrict__ x, int npix, int C, int xp, long long xplane, double* __restrict__ stats) {
  const int groups = C / 8;
  const int b = blockIdx.y;
  const int g = threadIdx.x % groups;           // blockDim.x is a multiple of groups
  const int lanes = blockDim.x / groups;        // pixels handled concurrently by the CTA
  const int pl = threadIdx.x / groups;
  const int chunk = (npix + gridDim.x - 1) / gridDim.x;
  const int p0 = blockIdx.x * chunk, p1 = min(npix, p0 + chunk);
  const float k = gn_pivot(x, b, g, npix, xp, xplane);
  double s = 0.0, ss = 0.0;
  float fs = 0.0f, fss = 0.0f;
  int cnt = 0;
  for (int p = p0 + pl; p < p1; p += lanes) {
    const size_t o = ((size_t)b * npix + p) * xp + g * 8;
    const uint4 hv = __ldg(reinterpret_cast<const uint4*>(x + o));
    const uint4 lv = __ldg(reinterpret_cast<const uint4*>(x + o + xplane));
    const uint32_t* hw = reinterpret_cast<const uint32_t*>(&hv);
    const uint32_t* lw = reinterpret_cast<const uint32_t*>(&lv);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hw[e]));
      const float2 lf = __half22float2(*reinterpret_cast<const __half2*>(&lw[e]));
      const float v0 = (hf.x + lf.x) - k, v1 = (hf.y + lf.y) - k;
      fs += v0 + v1;
      fss += v0 * v0 + v1 * v1;
    }
    if (++cnt == 8) {
      s += fs;
      ss += fss;
      fs = fss = 0.0f;
      cnt = 0;
    }
  }
  s += fs;
  ss += fss;
  atomicAdd(&stats[((size_t)b * groups + g) * 2 + 0], s);
  atomicAdd(&stats[((size_t)b * groups + g) * 2 + 1], ss);
}

// pass 2: y = relu((x - mean) * rstd * gamma + beta), re-split to hi/lo
__global__ void gn_apply_kernel(const __half* __restrict__ x, int npix, int C, int xp, long long xplane, const double* __restrict__ stats,
                                const float* __restrict__ gamma, const float* __restrict__ beta, float eps, int relu,
                                __half* __restrict__ y, int yp, long long yplane) {
  const int groups = C / 8;
  const int b = blockIdx.y;
  const long long n = (long long)npix * groups;
  const double inv_n = 1.0 / ((double)npix * 8.0);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int g = (int)(i % groups);
    const long long p = i / groups;
    const double d = stats[((size_t)b * groups + g) * 2] * inv_n;  // mean - pivot
    const double var = fmax(stats[((size_t)b * groups + g) * 2 + 1] * inv_n - d * d, 0.0);
    const float mean = (float)((double)gn_pivot(x, b, g, npix, xp, xplane) + d), rstd = (float)(1.0 / sqrt(var + (double)eps));
    const size_t o = ((size_t)b * npix + p) * xp + g * 8;
    const uint4 hv = __ldg(reinterpret_cast<const uint4*>(x + o));
    const uint4 lv = __ldg(reinterpret_cast<const uint4*>(x + o + xplane));
    const uint32_t* hw = reinterpret_cast<const uint32_t*>(&hv);
    const uint32_t* lw = reinterpret_cast<const uint32_t*>(&lv);
    uint32_t oh[4], ol[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hw[e]));
      const float2 lf = __half22float2(*reinterpret_cast<const __half2*>(&lw[e]));
      float v0 = ((hf.x + lf.x) - mean) * rstd * __ldg(gamma + g * 8 + 2 * e) + __ldg(beta + g * 8 + 2 * e);
      float v1 = ((hf.y + lf.y) - mean) * rstd * __ldg(gamma + g * 8 + 2 * e + 1) + __ldg(beta + g * 8 + 2 * e + 1);
      if (relu) {
        v0 = fmaxf(v0, 0.0f);
        v1 = fmaxf(v1, 0.0f);
      }
      split_pair(v0, v1, oh[e], ol[e]);
    }
    const size_t oo = ((size_t)b * npix + p) * yp + g * 8;
    *reinterpret_cast<uint4*>(y + oo) = make_uint4(oh[0], oh[1], oh[2], oh[3]);
    *reinterpret_cast<uint4*>(y + oo + yplane) = make_uint4(ol[0], ol[1], ol[2], ol[3]);
  }
}

// ------------------------------------------------------------------ depthwise 3x3 conv (+folded BN bias, ReLU), dilated
// One thread per (output pixel, 8-channel vector): 9 taps x (hi, lo) 16-byte loads, fp32 accumulate, hi/lo split on store.
// weights: fp32 [9][C] (tap-major, BN scale folded), bias fp32 [C].  HBM/L2-bound (AI ~ 2 flop/B): no tensor cores.
// Work decomposition: CTA = 8 x 8 output pixels x four 8-channel vectors (64 contiguous bytes per pixel and plane, i.e. whole 32-byte
// sectors); grid (pixel tiles, channel slabs, B) -- 32-bit index math only, and the nine taps of neighbouring pixels are requested
// by the same CTA at about the same time, so the halo re-reads hit L1 instead of going back to L2 nine times.
__global__ void __launch_bounds__(256) dwconv3x3_kernel(const __half* __restrict__ x, int H, int W, int C, int xp, long long xplane,
                                                        const float* __restrict__ wgt, const float* __restrict__ bias, int dil, int relu,
                                                        __half* __restrict__ y, int yp, long long yplane, int tiles_x) {
  const int cvec = threadIdx.x & 3, px = (threadIdx.x >> 2) & 7, py = threadIdx.x >> 5;
  const int tx = blockIdx.x % tiles_x, ty = blockIdx.x / tiles_x;
  const int w = tx * 8 + px, h = ty * 8 + py;
  const int c8 = blockIdx.y * 4 + cvec;
  const int b = blockIdx.z;
  if (w >= W || h >= H || c8 * 8 >= C) return;
  {
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = __ldg(bias + c8 * 8 + k);
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const int hh = h + (ky - 1) * dil;
      if (hh < 0 || hh >= H) continue;
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int ww = w + (kx - 1) * dil;
        if (ww < 0 || ww >= W) continue;
        const size_t o = (((size_t)b * H + hh) * W + ww) * xp + c8 * 8;
        const uint4 hv = __ldg(reinterpret_cast<const uint4*>(x + o));
        const uint4 lv = __ldg(reinterpret_cast<const uint4*>(x + o + xplane));
        const float4 w0 = __ldg(reinterpret_cast<const float4*>(wgt + (ky * 3 + kx) * C + c8 * 8));
        const float4 w1 = __ldg(reinterpret_cast<const float4*>(wgt + (ky * 3 + kx) * C + c8 * 8 + 4));
        const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
        const uint32_t* hw = reinterpret_cast<const uint32_t*>(&hv);
        const uint32_t* lw = reinterpret_cast<const uint32_t*>(&lv);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hw[e]));
          const float2 lf = __half22float2(*reinterpret_cast<const __half2*>(&lw[e]));
          acc[2 * e] = fmaf(hf.x + lf.x, wv[2 * e], acc[2 * e]);
          acc[2 * e + 1] = fmaf(hf.y + lf.y, wv[2 * e + 1], acc[2 * e + 1]);
        }
      }
    }
    uint32_t oh[4], ol[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      float v0 = acc[2 * e], v1 = acc[2 * e + 1];
      if (relu) {
        v0 = fmaxf(v0, 0.0f);
        v1 = fmaxf(v1, 0.0f);
      }
      split_pair(v0, v1, oh[e], ol[e]);
    }
    const size_t oo = (((size_t)b * H + h) * W + w) * yp + c8 * 8;
    *reinterpret_cast<uint4*>(y + oo) = make_uint4(oh[0], oh[1], oh[2], oh[3]);
    *reinterpret_cast<uint4*>(y + oo + yplane) = make_uint4(ol[0], ol[1], ol[2], ol[3]);
  }
}

// dilation 1 specialisation: one thread produces FOUR horizontally adjacent output pixels of one 8-channel vector.  The 3 x 6 input
// window is loaded once (36 instead of 72 vector loads) and the 72 filter taps stay in registers (18 loads per four pixels instead
// of 72): the kernel is bound by L1 bandwidth / issue slots, not by HBM, so fewer loads per output is what counts
// (5.1 -> 2.x ms for the 576-channel 256x512 DeepLab decoder layer).  Same fp32 accumulation order per output as the generic kernel
// (taps in (ky, kx) order), hence bit-identical results.
__global__ void __launch_bounds__(256) dwconv3x3_d1_kernel(const __half* __restrict__ x, int H, int W, int C, int xp, long long xplane,
                                                           const float* __restrict__ wgt, const float* __restrict__ bias, int relu,
                                                           __half* __restrict__ y, int yp, long long yplane, int tiles_x) {
  const int cvec = threadIdx.x & 3, pg = (threadIdx.x >> 2) & 7, py = threadIdx.x >> 5;
  // grid (pixel tiles, channel slabs, B).  (Making the channel slab the fastest-varying CTA index -- co-running CTAs covering whole
  // pixel rows -- measured 25 % SLOWER: 4.3 -> 5.5 ms on the 576-channel decoder layer.)
  const int tx = blockIdx.x % tiles_x, ty = blockIdx.x / tiles_x;
  const int w0 = tx * 32 + pg * 4, h = ty * 8 + py;
  const int c8 = blockIdx.y * 4 + cvec;
  const int b = blockIdx.z;

  if (w0 >= W || h >= H || c8 * 8 >= C) return;
  float wv[9][8];
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(wgt + t * C + c8 * 8));
    const float4 c = __ldg(reinterpret_cast<const float4*>(wgt + t * C + c8 * 8 + 4));
    wv[t][0] = a.x, wv[t][1] = a.y, wv[t][2] = a.z, wv[t][3] = a.w, wv[t][4] = c.x, wv[t][5] = c.y, wv[t][6] = c.z, wv[t][7] = c.w;
  }
  float acc[4][8];
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[j][k] = __ldg(bias + c8 * 8 + k);
#pragma unroll
  for (int ky = 0; ky < 3; ++ky) {
    const int hh = h + ky - 1;
    if (hh < 0 || hh >= H) continue;
    const __half* row = x + (((size_t)b * H + hh) * W) * xp + c8 * 8;
    // per output pixel the taps must be accumulated in kx order 0, 1, 2: walk the window columns left to right
#pragma unroll
    for (int cc = 0; cc < 6; ++cc) {
      const int ww = w0 + cc - 1;
      if (ww < 0 || ww >= W) continue;
      const uint4 hv = __ldg(reinterpret_cast<const uint4*>(row + (size_t)ww * xp));
      const uint4 lv = __ldg(reinterpret_cast<const uint4*>(row + (size_t)ww * xp + xplane));
      const uint32_t* hw = reinterpret_cast<const uint32_t*>(&hv);
      const uint32_t* lw = reinterpret_cast<const uint32_t*>(&lv);
      float v[8];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hw[e]));
        const float2 lf = __half22float2(*reinterpret_cast<const __half2*>(&lw[e]));
        v[2 * e] = hf.x + lf.x;
        v[2 * e + 1] = hf.y + lf.y;
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int kx = cc - j;  // window column cc is tap kx of output pixel j
        if (kx >= 0 && kx <= 2) {
#pragma unroll
          for (int k = 0; k < 8; ++k) acc[j][k] = fmaf(v[k], wv[ky * 3 + kx][k], acc[j][k]);
        }
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    if (w0 + j >= W) break;
    uint32_t oh[4], ol[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      float v0 = acc[j][2 * e], v1 = acc[j][2 * e + 1];
      if (relu) {
        v0 = fmaxf(v0, 0.0f);
        v1 = fmaxf(v1, 0.0f);
      }
      split_pair(v0, v1, oh[e], ol[e]);
    }
    const size_t oo = (((size_t)b * H + h) * W + (w0 + j)) * yp + c8 * 8;
    *reinterpret_cast<uint4*>(y + oo) = make_uint4(oh[0], oh[1], oh[2], oh[3]);
    *reinterpret_cast<uint4*>(y + oo + yplane) = make_uint4(ol[0], ol[1], ol[2], ol[3]);
  }
}

// ------------------------------------------------------------------ global average pool -> [B,1,1,C]
__global__ void global_avgpool_kernel(const __half* __restrict__ x, int npix, int C, int xp, long long xplane, __half* __restrict__ y,
                                      int yp, long long yplane) {
  // grid (C/8, B), block 256: each thread strides over pixels for one 8-channel vector; block reduce
  __shared__ float red[8][256];
  const int c8 = blockIdx.x, b = blockIdx.y;
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int p = threadIdx.x; p < npix; p += blockDim.x) {
    const size_t o = ((size_t)b * npix + p) * xp + c8 * 8;
    const uint4 hv = __ldg(reinterpret_cast<const uint4*>(x + o));
    const uint4 lv = __ldg(reinterpret_cast<const uint4*>(x + o + xplane));
    const uint32_t* hw = reinterpret_cast<const uint32_t*>(&hv);
    const uint32_t* lw = reinterpret_cast<const uint32_t*>(&lv);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hw[e]));
      const float2 lf = __half22float2(*reinterpret_cast<const __half2*>(&lw[e]));
      acc[2 * e] += hf.x + lf.x;
      acc[2 * e + 1] += hf.y + lf.y;
    }
  }
#pragma unroll
  for (int k = 0; k < 8; ++k) red[k][threadIdx.x] = acc[k];
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s)
#pragma unroll
      for (int k = 0; k < 8; ++k) red[k][threadIdx.x] += red[k][threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x < 8) {
    const float m = red[threadIdx.x][0] / (float)npix;
    uint32_t h, l;
    split_pair(m, m, h, l);
    y[(size_t)b * yp + c8 * 8 + threadIdx.x] = __ushort_as_half((unsigned short)h);
    y[(size_t)b * yp + c8 * 8 + threadIdx.x + yplane] = __ushort_as_half((unsigned short)l);
  }
}

// ------------------------------------------------------------------ bilinear resize (align_corners = False), split16 -> split16
// CTA = 8 x 8 output pixels x four 8-channel vectors, grid (pixel tiles, channel slabs, B): 32-bit index math, 64-byte runs per pixel.
__global__ void __launch_bounds__(256) bilinear_resize_kernel(const __half* __restrict__ x, int Hi, int Wi, int C, int xp, long long xplane,
                                                              __half* __restrict__ y, int Ho, int Wo, int yp, long long yplane, int tiles_x) {
  const int cvec = threadIdx.x & 3, px = (threadIdx.x >> 2) & 7, py = threadIdx.x >> 5;
  const int tx = blockIdx.x % tiles_x, ty = blockIdx.x / tiles_x;
  const int wo = tx * 8 + px, ho = ty * 8 + py;
  const int c8 = blockIdx.y * 4 + cvec;
  const int b = blockIdx.z;
  if (wo >= Wo || ho >= Ho || c8 * 8 >= C) return;
  const float sh = (float)Hi / (float)Ho, sw = (float)Wi / (float)Wo;
  {
    int h0, h1, w0, w1;
    float lh, lw_;
    bilinear_src(ho, sh, Hi, &h0, &h1, &lh);
    bilinear_src(wo, sw, Wi, &w0, &w1, &lw_);
    const float wgt[4] = {(1.0f - lh) * (1.0f - lw_), (1.0f - lh) * lw_, lh * (1.0f - lw_), lh * lw_};
    const int hs[4] = {h0, h0, h1, h1}, ws[4] = {w0, w1, w0, w1};
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const size_t o = (((size_t)b * Hi + hs[k]) * Wi + ws[k]) * xp + c8 * 8;
      const uint4 hv = __ldg(reinterpret_cast<const uint4*>(x + o));
      const uint4 lv = __ldg(reinterpret_cast<const uint4*>(x + o + xplane));
      const uint32_t* hw = reinterpret_cast<const uint32_t*>(&hv);
      const uint32_t* lw = reinterpret_cast<const uint32_t*>(&lv);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hw[e]));
        const float2 lf = __half22float2(*reinterpret_cast<const __half2*>(&lw[e]));
        acc[2 * e] = fmaf(hf.x + lf.x, wgt[k], acc[2 * e]);
        acc[2 * e + 1] = fmaf(hf.y + lf.y, wgt[k], acc[2 * e + 1]);
      }
    }
    uint32_t oh[4], ol[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      split_pair(acc[2 * e], acc[2 * e + 1], oh[e], ol[e]);
    }
    const size_t oo = (((size_t)b * Ho + ho) * Wo + wo) * yp + c8 * 8;
    *reinterpret_cast<uint4*>(y + oo) = make_uint4(oh[0], oh[1], oh[2], oh[3]);
    *reinterpret_cast<uint4*>(y + oo + yplane) = make_uint4(ol[0], ol[1], ol[2], ol[3]);
  }
}

// ------------------------------------------------------------------ fused bilinear upsample + argmax over classes
// logits fp32 NHWC [B,hi,wi,pitch>=nc] -> labels int64 [B,Ho,Wo].  The [B,nc,Ho,Wo] fp32 tensor the reference materialises
// (2.55 GB at 16x19x1024x2048, segmentors/encoder_decoder.py:132-133) never exists.  First maximum wins (torch.argmax).
// Grid (ceil(Wo / 256), Ho, B), one output pixel per thread, 32-bit index math; the four corner logit rows are read as float4
// (rows are 16-byte aligned: pitch % 4 == 0), four classes per step, compared in class order.
__global__ void __launch_bounds__(256) upsample_argmax_kernel(const float* __restrict__ lg, int Hi, int Wi, int pitch, int nc,
                                                              long long* __restrict__ out, int Ho, int Wo) {
  const int wo = blockIdx.x * 256 + threadIdx.x;
  const int ho = blockIdx.y, b = blockIdx.z;
  if (wo >= Wo) return;
  const float sh = (float)Hi / (float)Ho, sw = (float)Wi / (float)Wo;
  int h0, h1, w0, w1;
  float lh, lw_;
  bilinear_src(ho, sh, Hi, &h0, &h1, &lh);
  bilinear_src(wo, sw, Wi, &w0, &w1, &lw_);
  const float* p00 = lg + (((size_t)b * Hi + h0) * Wi + w0) * pitch;
  const float* p01 = lg + (((size_t)b * Hi + h0) * Wi + w1) * pitch;
  const float* p10 = lg + (((size_t)b * Hi + h1) * Wi + w0) * pitch;
  const float* p11 = lg + (((size_t)b * Hi + h1) * Wi + w1) * pitch;
  const float a00 = (1.0f - lh) * (1.0f - lw_), a01 = (1.0f - lh) * lw_, a10 = lh * (1.0f - lw_), a11 = lh * lw_;
  float best = -CUDART_INF_F;
  int bi = 0;
  for (int c = 0; c < nc; c += 4) {
    const float4 q00 = __ldg(reinterpret_cast<const float4*>(p00 + c)), q01 = __ldg(reinterpret_cast<const float4*>(p01 + c));
    const float4 q10 = __ldg(reinterpret_cast<const float4*>(p10 + c)), q11 = __ldg(reinterpret_cast<const float4*>(p11 + c));
    const float v[4] = {a00 * q00.x + a01 * q01.x + a10 * q10.x + a11 * q11.x, a00 * q00.y + a01 * q01.y + a10 * q10.y + a11 * q11.y,
                        a00 * q00.z + a01 * q01.z + a10 * q10.z + a11 * q11.z, a00 * q00.w + a01 * q01.w + a10 * q10.w + a11 * q11.w};
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (c + k < nc && v[k] > best) {
        best = v[k];
        bi = c + k;
      }
  }
  out[((size_t)b * Ho + ho) * Wo + wo] = (long long)bi;
}

// ------------------------------------------------------------------ output side (SURVEY.md 8 f-2)
// Detection rows back to original-image coordinates, in place, for the first count[b] rows of every image:
//   x -= pad[1]; y -= pad[0]; x /= scale[1]; y /= scale[0]; clip to [0, width] / [0, height]     (src/models/yolov5.py:274-281,
//   src/models/yolox.py:171-178, src/models/fcos.py:150-161) -- fp32 subtract / IEEE divide / min-max like the numpy lines.
__global__ void rescale_clip_boxes_kernel(float* __restrict__ rows, int M, int row_stride, const int* __restrict__ count,
                                          const float* __restrict__ pads, const float* __restrict__ scales, const float* __restrict__ wh) {
  const int b = blockIdx.y;
  const int n = min(count[b], M);
  const float p0 = pads[b * 2], p1 = pads[b * 2 + 1], s0 = scales[b * 2], s1 = scales[b * 2 + 1], w = wh[b * 2], h = wh[b * 2 + 1];
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < n; r += gridDim.x * blockDim.x) {
    float* q = rows + ((size_t)b * M + r) * row_stride;
    const float x1 = __fdiv_rn(__fsub_rn(q[0], p1), s1), y1 = __fdiv_rn(__fsub_rn(q[1], p0), s0);
    const float x2 = __fdiv_rn(__fsub_rn(q[2], p1), s1), y2 = __fdiv_rn(__fsub_rn(q[3], p0), s0);
    q[0] = fminf(fmaxf(x1, 0.0f), w);
    q[1] = fminf(fmaxf(y1, 0.0f), h);
    q[2] = fminf(fmaxf(x2, 0.0f), w);
    q[3] = fminf(fmaxf(y2, 0.0f), h);
  }
}

// Segmentation confusion matrix (src/evaluator/eval_segmentation.py:52-57): cm[gt * nc + pred] += 1 for every pixel with
// 0 <= gt < nc.  Shared-memory privatised counters per CTA (nc <= 64), flushed with 64-bit global atomics.
__global__ void __launch_bounds__(256) confusion_matrix_kernel(const long long* __restrict__ gt, const long long* __restrict__ pred, long long n,
                                                               int nc, unsigned long long* __restrict__ cm) {
  extern __shared__ uint32_t s_cm[];
  const int bins = nc * nc;
  for (int i = threadIdx.x; i < bins; i += blockDim.x) s_cm[i] = 0;
  __syncthreads();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long g = gt[i];
    if (g >= 0 && g < nc) {
      const long long p = pred[i];
      if (p >= 0 && p < nc) atomicAdd(&s_cm[(int)g * nc + (int)p], 1u);  // np.bincount would raise on p outside [0, nc): not counted here
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < bins; i += blockDim.x) {
    const uint32_t c = s_cm[i];
    if (c) atomicAdd(&cm[i], (unsigned long long)c);
  }
}

static int check_split_view(const CvbView* v, const char* what) {
  CVB_REQUIRE(v != nullptr && v->base != nullptr, "%s: null view", what);
  CVB_REQUIRE(v->c_pitch >= v->C && v->plane_stride % 2 == 0, "%s: bad view", what);
  return CVB_OK;
}

}  // namespace cvb

using namespace cvb;

extern "C" int cvb_nchw_to_split(const float* src, int32_t B, int32_t C, int32_t H, int32_t W, const CvbView* dst, void* stream) {
  int rc = check_split_view(dst, "nchw_to_split");
  if (rc) return rc;
  CVB_REQUIRE(src && dst->B == B && dst->C == C && dst->H == H && dst->W == W, "nchw_to_split: shape mismatch");
  CVB_REQUIRE((long long)B * H < 0x7fffffffLL, "nchw_to_split: too many image rows");
  for (int bh0 = 0; bh0 < B * H; bh0 += kMaxGridZ) {
    dim3 grid(ceil_div(W, 32), ceil_div(C, 32), min(B * H - bh0, kMaxGridZ)), block(32, 8);
    nchw_to_split_kernel<<<grid, block, 0, as_stream(stream)>>>(src, B, C, H, W, static_cast<__half*>(dst->base), dst->c_pitch,
                                                                dst->plane_stride / 2, bh0);
    CVB_CHECK_CUDA(cudaGetLastError());
    count_launch();
  }
  return CVB_OK;
}

extern "C" int cvb_split_to_nchw(const CvbView* src, float* dst, void* stream) {
  int rc = check_split_view(src, "split_to_nchw");
  if (rc) return rc;
  CVB_REQUIRE(dst != nullptr, "split_to_nchw: null dst");
  CVB_REQUIRE((long long)src->B * src->H < 0x7fffffffLL, "split_to_nchw: too many image rows");
  const int rows = src->B * src->H;
  for (int bh0 = 0; bh0 < rows; bh0 += kMaxGridZ) {
    dim3 grid(ceil_div(src->W, 32), ceil_div(src->C, 32), min(rows - bh0, kMaxGridZ)), block(32, 8);
    split_to_nchw_kernel<<<grid, block, 0, as_stream(stream)>>>(static_cast<const __half*>(src->base), src->B, src->C, src->H, src->W,
                                                                src->c_pitch, src->plane_stride / 2, dst, bh0);
    CVB_CHECK_CUDA(cudaGetLastError());
    count_launch();
  }
  return CVB_OK;
}

extern "C" int cvb_f32nhwc_to_nchw(const CvbView* src, float* dst, void* stream) {
  CVB_REQUIRE(src && src->base && dst, "f32nhwc_to_nchw: null argument");
  CVB_REQUIRE((long long)src->B * src->H < 0x7fffffffLL, "f32nhwc_to_nchw: too many image rows");
  const int rows = src->B * src->H;
  for (int bh0 = 0; bh0 < rows; bh0 += kMaxGridZ) {
    dim3 grid(ceil_div(src->W, 32), ceil_div(src->C, 32), min(rows - bh0, kMaxGridZ)), block(32, 8);
    f32nhwc_to_nchw_kernel<<<grid, block, 0, as_stream(stream)>>>(static_cast<const float*>(src->base), src->B, src->C, src->H, src->W,
                                                                  src->c_pitch, dst, bh0);
    CVB_CHECK_CUDA(cudaGetLastError());
    count_launch();
  }
  return CVB_OK;
}

extern "C" int cvb_stem_s2d(const float* src, int32_t B, int32_t H, int32_t W, const CvbView* dst, int32_t pad_left, void* stream) {
  int rc = check_split_view(dst, "stem_s2d");
  if (rc) return rc;
  CVB_REQUIRE(src && H % 2 == 0 && W % 2 == 0, "stem_s2d: H and W must be even");
  CVB_REQUIRE(dst->B == B && dst->H == H / 2 && dst->W >= W / 2 + pad_left && pad_left >= 0 && dst->C == 16 && dst->c_pitch == 16,
              "stem_s2d: dst must be [B,H/2,>=W/2+pad_left,16]");
  CVB_REQUIRE(is_aligned(src, 8) && is_aligned(dst->base, 16) && dst->plane_stride % 16 == 0,
              "stem_s2d: alignment");
  const long long n = (long long)B * (H / 2) * (W / 2);
  const int block = 256;
  long long grid = (n + block - 1) / block;
  if (grid > kSmCount * 32) grid = kSmCount * 32;
  stem_s2d_kernel<<<(int)grid, block, 0, as_stream(stream)>>>(src, B, H, W, static_cast<__half*>(dst->base), dst->c_pitch,
                                                             dst->plane_stride / 2, dst->W, pad_left);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}

extern "C" int cvb_stem_s2d_u8(const uint8_t* src, int32_t B, int32_t H, int32_t W, const float* mean, const float* std, int32_t reverse_channels,
                               const CvbView* dst, int32_t pad_left, void* stream) {
  int rc = check_split_view(dst, "stem_s2d_u8");
  if (rc) return rc;
  CVB_REQUIRE(src && mean && std && H % 2 == 0 && W % 2 == 0, "stem_s2d_u8: null argument or odd H/W");
  CVB_REQUIRE(std[0] != 0.0f && std[1] != 0.0f && std[2] != 0.0f, "stem_s2d_u8: zero std");
  CVB_REQUIRE(dst->B == B && dst->H == H / 2 && dst->W >= W / 2 + pad_left && pad_left >= 0 && dst->C == 16 && dst->c_pitch == 16,
              "stem_s2d_u8: dst must be [B,H/2,>=W/2+pad_left,16]");
  CVB_REQUIRE(is_aligned(src, 2) && is_aligned(dst->base, 16) && dst->plane_stride % 16 == 0,
              "stem_s2d_u8: alignment");
  const bool pair = (W % 4 == 0) && is_aligned(src, 4);
  const long long n = (long long)B * (H / 2) * (W / 2) / (pair ? 2 : 1);
  const int block = 256;
  long long grid = (n + block - 1) / block;
  if (grid > kSmCount * 16) grid = kSmCount * 16;
  __half* dp = static_cast<__half*>(dst->base);
  if (pair)
    stem_s2d_u8_kernel<true><<<(int)grid, block, 0, as_stream(stream)>>>(src, B, H, W, mean[0], mean[1], mean[2], std[0], std[1], std[2],
                                                                        reverse_channels, dp, dst->c_pitch, dst->plane_stride / 2, dst->W, pad_left);
  else
    stem_s2d_u8_kernel<false><<<(int)grid, block, 0, as_stream(stream)>>>(src, B, H, W, mean[0], mean[1], mean[2], std[0], std[1], std[2],
                                                                         reverse_channels, dp, dst->c_pitch, dst->plane_stride / 2, dst->W, pad_left);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}

extern "C" int cvb_sppf_pool(const CvbView* x, const CvbView* y1, const CvbView* y2, const CvbView* y3, void* stream) {
  int rc = check_split_view(x, "sppf x");
  if (!rc) rc = check_split_view(y1, "sppf y1");
  if (!rc) rc = check_split_view(y2, "sppf y2");
  if (!rc) rc = check_split_view(y3, "sppf y3");
  if (rc) return rc;
  const CvbView* vs[4] = {x, y1, y2, y3};
  for (int i = 0; i < 4; ++i) {
    CVB_REQUIRE(vs[i]->B == x->B && vs[i]->H == x->H && vs[i]->W == x->W && vs[i]->C == x->C, "sppf: view %d shape mismatch", i);
    CVB_REQUIRE(vs[i]->c_pitch % 8 == 0 && is_aligned(vs[i]->base, 16) && vs[i]->plane_stride % 16 == 0,
                "sppf: view %d alignment", i);
  }
  CVB_REQUIRE(x->C % 8 == 0, "sppf: C must be a multiple of 8");
  const size_t smem = (size_t)x->H * x->W * 8 * sizeof(float) * 2;
  CVB_REQUIRE(smem <= 200 * 1024, "sppf: map %dx%d too large for the shared-memory pool kernel", x->H, x->W);
  // one-time, thread-safe (C++11 static initialisation) opt-in to the large dynamic shared memory carve-out
  static const cudaError_t attr_set_err = opt_in_smem(sppf_pool_kernel, 200 * 1024);
  CVB_CHECK_CUDA(attr_set_err);
  const int cgroups = x->C / 8;
  sppf_pool_kernel<<<x->B * cgroups, 256, smem, as_stream(stream)>>>(
      static_cast<const __half*>(x->base), x->H, x->W, x->c_pitch, x->plane_stride / 2, static_cast<__half*>(y1->base), y1->c_pitch,
      y1->plane_stride / 2, static_cast<__half*>(y2->base), y2->c_pitch, y2->plane_stride / 2, static_cast<__half*>(y3->base), y3->c_pitch,
      y3->plane_stride / 2, cgroups);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}

// What both decode entry points launch: K<HIST, MULTI> with HIST iff there is an NMS workspace and MULTI iff multi_label with nc > 1
// (the rule of cvb_yolo_nms), the workspace's histograms and rowmax, and the shared-memory histogram of HIST, to which both HIST
// instantiations are opted in once (thread-safe static initialisation).
template <auto kPlain, auto kSingle, auto kMulti>
static int decode_prepass(void* ws, int B, bool multi, decltype(kPlain)* kernel, uint32_t** hist, float** rowmax, size_t* smem) {
  static const cudaError_t single_smem_err = opt_in_smem(kSingle, kNmsBins * (int)sizeof(uint32_t));
  static const cudaError_t multi_smem_err = opt_in_smem(kMulti, kNmsBins * (int)sizeof(uint32_t));
  CVB_CHECK_CUDA(single_smem_err);
  CVB_CHECK_CUDA(multi_smem_err);
  *kernel = !ws ? kPlain : multi ? kMulti : kSingle;
  *hist = static_cast<uint32_t*>(ws);
  *rowmax = nms_ws_rowmax(ws, B);
  *smem = ws ? (size_t)kNmsBins * sizeof(uint32_t) : 0;
  return CVB_OK;
}

extern "C" int cvb_yolo_decode(const CvbView* raw, int32_t na, int32_t no, const float* anchors_px, float stride, float* z, int64_t z_rows,
                               int64_t z_off, float* xperm, void* nms_workspace, float conf_thres, int32_t multi_label, void* stream) {
  CVB_REQUIRE(raw && raw->base && anchors_px, "yolo_decode: null argument");
  CVB_REQUIRE(raw->c_pitch >= na * no, "yolo_decode: raw pitch %d < na*no %d", raw->c_pitch, na * no);
  CVB_REQUIRE(z != nullptr || xperm != nullptr, "yolo_decode: nothing to write");
  CVB_REQUIRE(nms_workspace == nullptr || z != nullptr, "yolo_decode: histogram needs the decoded output");
  CVB_REQUIRE((long long)raw->H * raw->W * na < 0x7fffffffLL, "yolo_decode: level too large");
  CVB_REQUIRE(no <= 96, "yolo_decode: at most 91 classes supported (no=%d)", no);
  if (int rc = z ? check_level_rows("yolo_decode", z_off, (long long)na * raw->H * raw->W, z_rows) : CVB_OK) return rc;
  auto kernel = yolo_decode_kernel<false, false>;
  uint32_t* hist;
  float* rowmax;
  size_t smem;
  if (int rc = decode_prepass<yolo_decode_kernel<false, false>, yolo_decode_kernel<true, false>, yolo_decode_kernel<true, true>>(
          nms_workspace, raw->B, multi_label && no - 5 > 1, &kernel, &hist, &rowmax, &smem))
    return rc;
  kernel<<<dim3(ceil_div(raw->H * raw->W, kDecodePix), raw->B), kDecodeThreads, smem, as_stream(stream)>>>(
      static_cast<const float*>(raw->base), raw->H, raw->W, raw->c_pitch, na, no, anchors_px, stride, z, z_rows, z_off, xperm, hist, rowmax,
      conf_thres, fast_div_magic(raw->W, (unsigned long long)raw->H * raw->W));
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}

extern "C" int cvb_yolov6_decode(const CvbView* cls, const CvbView* reg, int32_t nc, float stride, float* z, int64_t z_rows, int64_t z_off,
                                 void* nms_workspace, float conf_thres, int32_t multi_label, void* stream) {
  CVB_REQUIRE(cls && cls->base && reg && reg->base && z, "yolov6_decode: null argument");
  CVB_REQUIRE(nc >= 1 && nc <= 91, "yolov6_decode: 1..91 classes supported (nc=%d)", nc);
  CVB_REQUIRE(cls->plane_stride == 0 && reg->plane_stride == 0, "yolov6_decode: cls and reg must be fp32 views");
  CVB_REQUIRE(cls->C >= nc && cls->c_pitch >= cls->C && reg->C >= 4 && reg->c_pitch >= reg->C, "yolov6_decode: cls needs >= nc and reg >= 4 channels");
  CVB_REQUIRE(cls->B == reg->B && cls->H == reg->H && cls->W == reg->W, "yolov6_decode: cls [%d,%d,%d] and reg [%d,%d,%d] differ", cls->B, cls->H,
              cls->W, reg->B, reg->H, reg->W);
  CVB_REQUIRE((long long)cls->H * cls->W < 0x7fffffffLL, "yolov6_decode: level too large");
  if (int rc = check_level_rows("yolov6_decode", z_off, (long long)cls->H * cls->W, z_rows)) return rc;
  auto kernel = yolov6_decode_kernel<false, false>;
  uint32_t* hist;
  float* rowmax;
  size_t smem;
  if (int rc = decode_prepass<yolov6_decode_kernel<false, false>, yolov6_decode_kernel<true, false>, yolov6_decode_kernel<true, true>>(
          nms_workspace, cls->B, multi_label && nc > 1, &kernel, &hist, &rowmax, &smem))
    return rc;
  kernel<<<dim3(ceil_div(cls->H * cls->W, kV6DecodePix), cls->B), kV6DecodeThreads, smem, as_stream(stream)>>>(
      static_cast<const float*>(cls->base), cls->c_pitch, static_cast<const float*>(reg->base), reg->c_pitch, cls->H, cls->W, nc, stride, z, z_rows,
      z_off, hist, rowmax, conf_thres);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}

extern "C" int cvb_depth_to_space2(const CvbView* src, const CvbView* dst, void* stream) {
  int rc = check_split_view(src, "depth_to_space2 src");
  if (!rc) rc = check_split_view(dst, "depth_to_space2 dst");
  if (rc) return rc;
  CVB_REQUIRE(src->plane_stride > 0 && dst->plane_stride > 0, "depth_to_space2: src and dst must be split16 views");
  CVB_REQUIRE(dst->C % 8 == 0 && src->C == 4 * dst->C, "depth_to_space2: src must have 4 x dst's channels (src %d, dst %d), a multiple of 8",
              src->C, dst->C);
  CVB_REQUIRE(src->B == dst->B && dst->H == 2 * src->H && dst->W == 2 * src->W, "depth_to_space2: dst [%d,%d,%d] is not src [%d,%d,%d] at twice the size",
              dst->B, dst->H, dst->W, src->B, src->H, src->W);
  CVB_REQUIRE(src->c_pitch % 8 == 0 && dst->c_pitch % 8 == 0 && is_aligned(src->base, 16) && is_aligned(dst->base, 16) &&
                  src->plane_stride % 16 == 0 && dst->plane_stride % 16 == 0,
              "depth_to_space2: alignment");
  const long long n = (long long)dst->B * dst->H * dst->W * (dst->C / 8);
  if (n == 0) return CVB_OK;
  long long grid = (n + 255) / 256;
  if (grid > kSmCount * 16) grid = kSmCount * 16;
  depth_to_space2_kernel<<<(int)grid, 256, 0, as_stream(stream)>>>(static_cast<const __half*>(src->base), src->c_pitch, src->plane_stride / 2, src->H,
                                                                   src->W, dst->C, static_cast<__half*>(dst->base), dst->c_pitch, dst->plane_stride / 2, n);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}

static int check_vec_view(const CvbView* v, const char* what) {
  int rc = check_split_view(v, what);
  if (rc) return rc;
  CVB_REQUIRE(v->C % 8 == 0 && v->c_pitch % 8 == 0 && is_aligned(v->base, 16) && v->plane_stride % 16 == 0,
              "%s: channels/pitch must be multiples of 8 and 16-byte aligned", what);
  return CVB_OK;
}

extern "C" int cvb_maxpool3x3s2(const CvbView* x, const CvbView* y, void* stream) {
  int rc = check_vec_view(x, "maxpool x");
  if (!rc) rc = check_vec_view(y, "maxpool y");
  if (rc) return rc;
  const int Ho = (x->H + 2 - 3) / 2 + 1, Wo = (x->W + 2 - 3) / 2 + 1;
  CVB_REQUIRE(y->B == x->B && y->H == Ho && y->W == Wo && y->C == x->C, "maxpool3x3s2: output must be [%d,%d,%d,%d]", x->B, Ho, Wo, x->C);
  const long long n = (long long)x->B * Ho * Wo * (x->C / 8);
  long long grid = (n + 255) / 256;
  if (grid > kSmCount * 32) grid = kSmCount * 32;
  maxpool3x3s2_kernel<<<(int)grid, 256, 0, as_stream(stream)>>>(static_cast<const __half*>(x->base), x->B, x->H, x->W, x->C, x->c_pitch,
                                                               x->plane_stride / 2, static_cast<__half*>(y->base), Ho, Wo, y->c_pitch,
                                                               y->plane_stride / 2);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}

extern "C" int cvb_split_to_f32nhwc(const CvbView* x, const CvbView* y, void* stream) {
  int rc = check_vec_view(x, "split_to_f32 x");
  if (rc) return rc;
  CVB_REQUIRE(y && y->base && y->B == x->B && y->H == x->H && y->W == x->W && y->C == x->C && y->c_pitch % 4 == 0 &&
                  is_aligned(y->base, 16),
              "split_to_f32: output view mismatch");
  const long long npix = (long long)x->B * x->H * x->W;
  long long grid = (npix * (x->C / 8) + 255) / 256;
  if (grid > kSmCount * 32) grid = kSmCount * 32;
  split_to_f32_kernel<<<(int)grid, 256, 0, as_stream(stream)>>>(static_cast<const __half*>(x->base), npix, x->C, x->c_pitch,
                                                               x->plane_stride / 2, static_cast<float*>(y->base), y->c_pitch);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}

extern "C" size_t cvb_groupnorm_workspace_bytes(int32_t B, int32_t groups) { return (size_t)B * groups * 2 * sizeof(double); }

extern "C" int cvb_groupnorm_relu(const CvbView* x, int32_t groups, const float* gamma, const float* beta, float eps, int32_t relu,
                                  const CvbView* y, void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_vec_view(x, "groupnorm x");
  if (!rc) rc = check_vec_view(y, "groupnorm y");
  if (rc) return rc;
  CVB_REQUIRE(gamma && beta && workspace, "groupnorm: null argument");
  CVB_REQUIRE(groups > 0 && x->C == groups * 8, "groupnorm: only 8 channels per group are supported (C=%d, groups=%d)", x->C, groups);
  CVB_REQUIRE(y->B == x->B && y->H == x->H && y->W == x->W && y->C == x->C, "groupnorm: output view mismatch");
  CVB_REQUIRE(workspace_bytes >= cvb_groupnorm_workspace_bytes(x->B, groups) && is_aligned(workspace, 8),
              "groupnorm: workspace too small / misaligned");
  cudaStream_t st = as_stream(stream);
  CVB_CHECK_CUDA(cudaMemsetAsync(workspace, 0, cvb_groupnorm_workspace_bytes(x->B, groups), st));
  const int npix = x->H * x->W;
  CVB_REQUIRE(groups <= 1024, "groupnorm: at most 1024 groups (one CTA thread per group), got %d", groups);
  const int threads = 256 / groups * groups > 0 ? (256 / groups) * groups : groups;
  int chunks = (npix + 255) / 256;
  if (chunks > kSmCount * 4) chunks = kSmCount * 4;
  if (chunks < 1) chunks = 1;
  gn_stats_kernel<<<dim3(chunks, x->B), threads, 0, st>>>(static_cast<const __half*>(x->base), npix, x->C, x->c_pitch, x->plane_stride / 2,
                                                         static_cast<double*>(workspace));
  long long g2 = ((long long)npix * groups + 255) / 256;
  if (g2 > kSmCount * 8) g2 = kSmCount * 8;
  gn_apply_kernel<<<dim3((int)g2, x->B), 256, 0, st>>>(static_cast<const __half*>(x->base), npix, x->C, x->c_pitch, x->plane_stride / 2,
                                                      static_cast<const double*>(workspace), gamma, beta, eps, relu,
                                                      static_cast<__half*>(y->base), y->c_pitch, y->plane_stride / 2);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch(2);
  return CVB_OK;
}

extern "C" int cvb_dwconv3x3(const CvbView* x, const float* weights, const float* bias, int32_t dilation, int32_t relu, const CvbView* y,
                             void* stream) {
  int rc = check_vec_view(x, "dwconv x");
  if (!rc) rc = check_vec_view(y, "dwconv y");
  if (rc) return rc;
  CVB_REQUIRE(weights && bias && dilation >= 1, "dwconv3x3: bad argument");
  CVB_REQUIRE(y->B == x->B && y->H == x->H && y->W == x->W && y->C == x->C, "dwconv3x3: output view mismatch (stride 1, 'same' padding)");
  CVB_REQUIRE(is_aligned(weights, 16), "dwconv3x3: weights must be 16-byte aligned");
  const int tiles_x = ceil_div(x->W, 8), tiles_y = ceil_div(x->H, 8);
  CVB_REQUIRE(x->B <= 65535 && ceil_div(x->C / 8, 4) <= 65535, "dwconv3x3: batch / channel count too large for the launch grid");
  if (dilation == 1) {
    const int tx32 = ceil_div(x->W, 32);
    dim3 g1(tx32 * tiles_y, ceil_div(x->C / 8, 4), x->B);
    dwconv3x3_d1_kernel<<<g1, 256, 0, as_stream(stream)>>>(static_cast<const __half*>(x->base), x->H, x->W, x->C, x->c_pitch, x->plane_stride / 2,
                                                          weights, bias, relu, static_cast<__half*>(y->base), y->c_pitch, y->plane_stride / 2, tx32);
    CVB_CHECK_CUDA(cudaGetLastError());
    count_launch();
    return CVB_OK;
  }
  dim3 grid(tiles_x * tiles_y, ceil_div(x->C / 8, 4), x->B);
  dwconv3x3_kernel<<<grid, 256, 0, as_stream(stream)>>>(static_cast<const __half*>(x->base), x->H, x->W, x->C, x->c_pitch, x->plane_stride / 2,
                                                       weights, bias, dilation, relu, static_cast<__half*>(y->base), y->c_pitch,
                                                       y->plane_stride / 2, tiles_x);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}

extern "C" int cvb_global_avgpool(const CvbView* x, const CvbView* y, void* stream) {
  int rc = check_vec_view(x, "avgpool x");
  if (!rc) rc = check_split_view(y, "avgpool y");
  if (rc) return rc;
  CVB_REQUIRE(y->B == x->B && y->H == 1 && y->W == 1 && y->C == x->C, "global_avgpool: output must be [B,1,1,C]");
  global_avgpool_kernel<<<dim3(x->C / 8, x->B), 256, 0, as_stream(stream)>>>(static_cast<const __half*>(x->base), x->H * x->W, x->C, x->c_pitch,
                                                                            x->plane_stride / 2, static_cast<__half*>(y->base), y->c_pitch,
                                                                            y->plane_stride / 2);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}

extern "C" int cvb_bilinear_resize(const CvbView* x, const CvbView* y, void* stream) {
  int rc = check_vec_view(x, "bilinear x");
  if (!rc) rc = check_vec_view(y, "bilinear y");
  if (rc) return rc;
  CVB_REQUIRE(y->B == x->B && y->C == x->C, "bilinear_resize: batch/channel mismatch");
  const int tiles_x = ceil_div(y->W, 8), tiles_y = ceil_div(y->H, 8);
  CVB_REQUIRE(y->B <= 65535 && ceil_div(y->C / 8, 4) <= 65535, "bilinear_resize: batch / channel count too large for the launch grid");
  dim3 grid(tiles_x * tiles_y, ceil_div(y->C / 8, 4), y->B);
  bilinear_resize_kernel<<<grid, 256, 0, as_stream(stream)>>>(static_cast<const __half*>(x->base), x->H, x->W, x->C, x->c_pitch, x->plane_stride / 2,
                                                             static_cast<__half*>(y->base), y->H, y->W, y->c_pitch, y->plane_stride / 2, tiles_x);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}

extern "C" int cvb_upsample_argmax(const CvbView* logits, int32_t nc, int64_t* labels, int32_t Ho, int32_t Wo, void* stream) {
  CVB_REQUIRE(logits && logits->base && labels && nc > 0 && logits->c_pitch >= nc && Ho > 0 && Wo > 0, "upsample_argmax: bad argument");
  CVB_REQUIRE(logits->c_pitch % 4 == 0 && is_aligned(logits->base, 16) && logits->c_pitch >= (nc + 3) / 4 * 4,
              "upsample_argmax: logits rows must be 16-byte aligned and padded to a multiple of 4 classes");
  CVB_REQUIRE(Ho <= 65535 && logits->B <= 65535, "upsample_argmax: output too tall / batch too large for the launch grid");
  dim3 grid(ceil_div(Wo, 256), Ho, logits->B);
  upsample_argmax_kernel<<<grid, 256, 0, as_stream(stream)>>>(static_cast<const float*>(logits->base), logits->H, logits->W, logits->c_pitch, nc,
                                                             reinterpret_cast<long long*>(labels), Ho, Wo);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}

extern "C" int cvb_rescale_clip_boxes(float* rows, int32_t B, int32_t M, int32_t row_stride, const int32_t* count, const float* pads,
                                      const float* scales, const float* wh, void* stream) {
  CVB_REQUIRE(rows && count && pads && scales && wh && B > 0 && M > 0 && row_stride >= 4, "rescale_clip_boxes: bad argument");
  CVB_REQUIRE(B <= 65535, "rescale_clip_boxes: batch too large for the launch grid");
  dim3 grid(ceil_div(M, 256) < 8 ? ceil_div(M, 256) : 8, B);
  rescale_clip_boxes_kernel<<<grid, 256, 0, as_stream(stream)>>>(rows, M, row_stride, count, pads, scales, wh);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}

extern "C" int cvb_confusion_matrix(const int64_t* gt, const int64_t* pred, int64_t n, int32_t num_classes, int64_t* cm, void* stream) {
  CVB_REQUIRE(gt && pred && cm && n >= 0 && num_classes > 0 && num_classes <= 64, "confusion_matrix: bad argument (num_classes <= 64)");
  if (n == 0) return CVB_OK;
  long long grid = (n + 256LL * 16 - 1) / (256LL * 16);
  if (grid > kSmCount * 8) grid = kSmCount * 8;
  confusion_matrix_kernel<<<(int)grid, 256, (size_t)num_classes * num_classes * sizeof(uint32_t), as_stream(stream)>>>(
      reinterpret_cast<const long long*>(gt), reinterpret_cast<const long long*>(pred), n, num_classes, reinterpret_cast<unsigned long long*>(cm));
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}

// ------------------------------------------------------------------------------------------------ input side: letterbox (SURVEY.md 8 f-1)
// Resize(keep_ratio=True) of the reference (src/data/transforms/det_transforms.py:162-198): cv2.resize(INTER_LINEAR) of the uint8 HWC
// frame to (oh, ow), then cv2.copyMakeBorder with a constant fill.  OpenCV's 8-bit bilinear kernel, restated (imgproc/resize.cpp):
// per axis fx = (float)((d + 0.5) * scale - 0.5) with scale = 1 / (dst / src) in double, s = floor(fx), fx -= s; columns zero fx at the
// borders, rows clip the index; 11-bit coefficients = round-to-nearest-even of (1 - fx) * 2048 and fx * 2048 in float; horizontal pass in
// int32, vertical pass (((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2) >> 2.  Bit-identical to cv2 4.x (oracle/io_oracle.py,
// tests/golden/letterbox.npz).  geom[b] = (h, w, oh, ow, top, left); one thread per output pixel.
namespace cvb {
__device__ __forceinline__ void lb_axis(int d, int dst, int src, bool zero_at_border, int* s0, int* s1, int* c0, int* c1) {
  const double scale = 1.0 / ((double)dst / (double)src);
  float f = (float)(((double)d + 0.5) * scale - 0.5);
  int s = (int)floorf(f);
  f -= (float)s;
  if (zero_at_border) {
    if (s < 0) {
      f = 0.0f;
      s = 0;
    }
    if (s >= src - 1) {
      f = 0.0f;
      s = src - 1;
    }
    *s0 = s;
    *s1 = min(s + 1, src - 1);
  } else {
    *s0 = min(max(s, 0), src - 1);
    *s1 = min(max(s + 1, 0), src - 1);
  }
  *c0 = __float2int_rn(__fmul_rn(__fsub_rn(1.0f, f), 2048.0f));
  *c1 = __float2int_rn(__fmul_rn(f, 2048.0f));
}

__global__ void __launch_bounds__(256) letterbox_u8_kernel(const uint8_t* const* __restrict__ src, const int* __restrict__ geom, int B, int OH,
                                                           int OW, int f0, int f1, int f2, uint8_t* __restrict__ dst) {
  const long long n = (long long)B * OH * OW;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(i % OW);
    const long long t = i / OW;
    const int y = (int)(t % OH);
    const int b = (int)(t / OH);
    const int* g = geom + b * 6;
    const int h = g[0], w = g[1], oh = g[2], ow = g[3], top = g[4], left = g[5];
    const int dy = y - top, dx = x - left;
    int r0 = f0, r1 = f1, r2 = f2;
    if (dy >= 0 && dy < oh && dx >= 0 && dx < ow) {
      const uint8_t* s = src[b];
      if (h == oh && w == ow) {  // the reference skips cv2.resize when the size is unchanged
        const uint8_t* p = s + ((size_t)dy * w + dx) * 3;
        r0 = p[0];
        r1 = p[1];
        r2 = p[2];
      } else {
        int x0, x1, a0, a1, y0, y1, b0, b1;
        lb_axis(dx, ow, w, true, &x0, &x1, &a0, &a1);
        lb_axis(dy, oh, h, false, &y0, &y1, &b0, &b1);
        const uint8_t* p00 = s + ((size_t)y0 * w + x0) * 3;
        const uint8_t* p01 = s + ((size_t)y0 * w + x1) * 3;
        const uint8_t* p10 = s + ((size_t)y1 * w + x0) * 3;
        const uint8_t* p11 = s + ((size_t)y1 * w + x1) * 3;
        int out[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const int h0 = (int)p00[c] * a0 + (int)p01[c] * a1;
          const int h1 = (int)p10[c] * a0 + (int)p11[c] * a1;
          const int v = (((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2;
          out[c] = min(max(v, 0), 255);
        }
        r0 = out[0];
        r1 = out[1];
        r2 = out[2];
      }
    }
    uint8_t* q = dst + (size_t)i * 3;
    q[0] = (uint8_t)r0;
    q[1] = (uint8_t)r1;
    q[2] = (uint8_t)r2;
  }
}

// ------------------------------------------------------------------------------------------------ output side: COCO records (SURVEY.md 8 f-2)
// prepare_for_coco_detection + convert_to_xywh (src/evaluator/eval_coco.py:87-111, 200-202): one record per kept detection,
// (image_id, category_id) and (x, y, xmax - xmin, ymax - ymin, score) -- same fp32 subtraction as the torch lines -- compacted over the
// batch in image order.  One CTA per image; its offset is the sum of the preceding counts.
__global__ void __launch_bounds__(128) coco_pack_kernel(const float* __restrict__ rows, int M, int row_stride, const int* __restrict__ count,
                                                        const long long* __restrict__ image_ids, const int* __restrict__ id2cat, int nc,
                                                        long long* __restrict__ rec_ids, float* __restrict__ rec_box, int* __restrict__ total) {
  __shared__ int off_s;
  const int b = blockIdx.x;
  if (threadIdx.x < 32) {
    int acc = 0;
    for (int i = threadIdx.x; i < b; i += 32) acc += min(max(count[i], 0), M);
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (threadIdx.x == 0) off_s = acc;
  }
  __syncthreads();
  const int off = off_s;
  const int k = min(max(count[b], 0), M);
  if (b == (int)gridDim.x - 1 && threadIdx.x == 0) *total = off + k;
  const long long img = image_ids[b];
  for (int j = threadIdx.x; j < k; j += blockDim.x) {
    const float* r = rows + ((size_t)b * M + j) * row_stride;
    const float x1 = r[0], y1 = r[1], x2 = r[2], y2 = r[3];
    int cls = (int)r[5];
    if (id2cat != nullptr && cls >= 0 && cls < nc) cls = id2cat[cls];
    const size_t o = (size_t)(off + j);
    rec_ids[o * 2 + 0] = img;
    rec_ids[o * 2 + 1] = cls;
    float* q = rec_box + o * 5;
    q[0] = x1;
    q[1] = y1;
    q[2] = __fsub_rn(x2, x1);
    q[3] = __fsub_rn(y2, y1);
    q[4] = r[4];
  }
}
}  // namespace cvb

extern "C" int cvb_letterbox_u8(const uint8_t* const* src_ptrs, const int32_t* geom, int32_t B, int32_t out_h, int32_t out_w, const int32_t* fill,
                                uint8_t* dst, void* stream) {
  using namespace cvb;
  CVB_REQUIRE(src_ptrs && geom && fill && dst && B > 0 && out_h > 0 && out_w > 0, "letterbox: bad argument");
  const long long n = (long long)B * out_h * out_w;
  long long grid = (n + 255) / 256;
  if (grid > kSmCount * 16) grid = kSmCount * 16;
  letterbox_u8_kernel<<<(int)grid, 256, 0, as_stream(stream)>>>(src_ptrs, geom, B, out_h, out_w, fill[0], fill[1], fill[2], dst);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}

extern "C" int cvb_coco_pack(const float* rows, int32_t B, int32_t M, int32_t row_stride, const int32_t* count, const int64_t* image_ids,
                             const int32_t* id2category, int32_t num_classes, int64_t* rec_ids, float* rec_box, int32_t* total, void* stream) {
  using namespace cvb;
  CVB_REQUIRE(rows && count && image_ids && rec_ids && rec_box && total && B > 0 && M > 0 && row_stride >= 6, "coco_pack: bad argument");
  coco_pack_kernel<<<B, 128, 0, as_stream(stream)>>>(rows, M, row_stride, count, reinterpret_cast<const long long*>(image_ids), id2category,
                                                     num_classes, reinterpret_cast<long long*>(rec_ids), rec_box, total);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}
