// The segmentation cross-entropy loss with the bilinear upsample to label size fused in (src/losses/seg/cross_entropy_loss.py
// CrossEntropyLoss2d behind EncoderDecoder.loss_forward's F.interpolate; restated in oracle/seg_loss_oracle.py), and its gradient with
// respect to the head output preds [B, C, h, w].  The upsampled logits z [B, C, H, W] and their softmax never reach HBM.
//
// Forward (cvb_train_seg_ce_fwd), stream-ordered, no host sync, CUDA-graph capturable:
//   1. seg_ce_fwd_kernel    one thread per label pixel (four per thread, a CTA covers 1024 consecutive pixels): the label, the C
//                           interpolated logits in class order with a running maximum and sum of exponentials, lse = m + log(sum) saved
//                           for the backward (the one fp32 value per pixel), and lse - z_y, the valid count and the out-of-range count
//                           added to fp64 per-CTA partials.
//   2. seg_ce_final_kernel  one CTA: the partials in a fixed order -> loss = loss_weight * (sum / n_valid) and record = (n_valid, n_bad).
// Backward (cvb_train_seg_ce_bwd): seg_ce_bwd_kernel, a gather.  A CTA owns a TI x TJ tile of preds (all classes) and walks the full-res
// footprint whose taps reach the tile, in blocks that fit shared memory.  Per block and class it recomputes G = s (softmax - onehot) from
// the saved lse, sums G along each footprint row into the tile's columns, then along the footprint columns into the tile's rows; the
// upsample's transpose is separable, so that is d preds.  Every gradient element is written by one thread with sums in a fixed order: no
// float atomics, runs and graph replays are bitwise identical.
//
// The taps are bilinear_src (internal.h), the index map of torch's upsample_bilinear2d; it is monotone, so the full-res rows (columns)
// whose taps include a preds row (column) are one contiguous range, found by binary search.
#include <limits.h>
#include <math.h>

#include "internal.h"

namespace cvb {
namespace {

constexpr int kCeNcMax = 1024;
constexpr int kCeThreads = 256;
constexpr int kCePix = 4;                 // forward: pixels per thread
constexpr int kCeFinalThreads = 256;
constexpr int kCeBlockPix = 4800;         // backward: full-res pixels of one footprint block in shared memory (36 x 132 at x4 and x8)
constexpr int kCeMaxTI = 32, kCeMaxTJ = 128;
constexpr int kCeMaxDim = 65535;
constexpr int kCeIgnore = -1, kCeBad = -2;

struct CeShape {
  int B, C, h, w, H, W;
  long long sb, sh, sw;  // label strides in elements
  long long ignore;
  float scale_h, scale_w;  // (float)h / H, (float)w / W
};

// class of a label (kCeIgnore for ignore_index, kCeBad outside [0, C))
template <typename T>
__device__ __forceinline__ int ce_target(const T* __restrict__ lab, const CeShape& S, int b, int Y, int X) {
  const long long v = (long long)lab[b * S.sb + Y * S.sh + X * S.sw];
  if (v == S.ignore) return kCeIgnore;
  return (v >= 0 && v < S.C) ? (int)v : kCeBad;
}

// The taps of one full-res pixel: row offsets (times w) and columns of the two source rows / columns and their weights.
struct Taps {
  int r0, r1, c0, c1;
  float lh0, lh1, lw0, lw1;
};

__device__ __forceinline__ Taps ce_taps(const CeShape& S, int Y, int X) {
  Taps t;
  int h0, h1, w0, w1;
  bilinear_src(Y, S.scale_h, S.h, &h0, &h1, &t.lh1);
  bilinear_src(X, S.scale_w, S.w, &w0, &w1, &t.lw1);
  t.r0 = h0 * S.w;
  t.r1 = h1 * S.w;
  t.c0 = w0;
  t.c1 = w1;
  t.lh0 = 1.0f - t.lh1;
  t.lw0 = 1.0f - t.lw1;
  return t;
}

// torch's upsample_bilinear2d: lh0 (lw0 x00 + lw1 x01) + lh1 (lw0 x10 + lw1 x11)
__device__ __forceinline__ float ce_interp(const float* __restrict__ p, int r0, int r1, int c0, int c1, float lh0, float lh1, float lw0, float lw1) {
  return lh0 * (lw0 * __ldg(p + r0 + c0) + lw1 * __ldg(p + r0 + c1)) + lh1 * (lw0 * __ldg(p + r1 + c0) + lw1 * __ldg(p + r1 + c1));
}

// --------------------------------------------------------------------------------------------------------------------------- forward
template <typename T>
__global__ void __launch_bounds__(kCeThreads) seg_ce_fwd_kernel(const float* __restrict__ x, const T* __restrict__ lab, CeShape S,
                                                                float* __restrict__ lse_out, double* __restrict__ partial) {
  __shared__ double red[kCeThreads / 32][3];
  const int HW = S.H * S.W, hw = S.h * S.w;
  const long long n = (long long)S.B * HW;
  double v[3] = {0.0, 0.0, 0.0};  // sum of lse - z_y, valid pixels, out-of-range labels
#pragma unroll 1
  for (int k = 0; k < kCePix; ++k) {
    const long long pl = ((long long)blockIdx.x * kCePix + k) * kCeThreads + threadIdx.x;
    if (pl >= n) break;
    const int p = (int)pl;
    const int b = p / HW, r = p - b * HW, Y = r / S.W, X = r - Y * S.W;
    const int t = ce_target(lab, S, b, Y, X);
    float lse = 0.0f;
    if (t == kCeBad) {
      v[2] += 1.0;
    } else if (t >= 0) {
      const Taps q = ce_taps(S, Y, X);
      const float* xc = x + (size_t)b * S.C * hw;
      // running maximum m and sum s of exp(z - m), one exponential per class; a NaN logit makes s NaN
      float m = -INFINITY, s = 0.0f, zy = 0.0f;
#pragma unroll 4
      for (int c = 0; c < S.C; ++c, xc += hw) {
        const float z = ce_interp(xc, q.r0, q.r1, q.c0, q.c1, q.lh0, q.lh1, q.lw0, q.lw1);
        const float d = z - m;
        const float e = expf(-fabsf(d));
        s = d > 0.0f ? fmaf(s, e, 1.0f) : s + e;
        m = fmaxf(m, z);
        zy = c == t ? z : zy;
      }
      lse = m + logf(s);
      v[0] += (double)(lse - zy);
      v[1] += 1.0;
    }
    lse_out[p] = lse;
  }
  block_sum<kCeThreads>(v, red);
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < 3; ++k) partial[(size_t)blockIdx.x * 3 + k] = v[k];
  }
}

__global__ void __launch_bounds__(kCeFinalThreads) seg_ce_final_kernel(const double* __restrict__ partial, int nblk, float loss_weight,
                                                                       float* __restrict__ loss, long long* __restrict__ record) {
  __shared__ double red[kCeFinalThreads / 32][3];
  double v[3] = {0.0, 0.0, 0.0};
  for (int i = threadIdx.x; i < nblk; i += kCeFinalThreads) {
    v[0] += partial[(size_t)i * 3];
    v[1] += partial[(size_t)i * 3 + 1];
    v[2] += partial[(size_t)i * 3 + 2];
  }
  block_sum<kCeFinalThreads>(v, red);
  if (threadIdx.x == 0) {
    const long long n_valid = (long long)v[1], n_bad = (long long)v[2];
    record[0] = n_valid;
    record[1] = n_bad;
    // the mean over valid pixels (0 / 0 = NaN when every pixel is ignored, as torch's 'mean'), then the weight, as the reference does;
    // a label outside [0, C) makes the loss NaN (torch raises there)
    loss[0] = n_bad ? __int_as_float(0x7fffffff) : loss_weight * (float)(v[0] / v[1]);
  }
}

// --------------------------------------------------------------------------------------------------------------------------- backward
struct CeTile {
  int TI, TJ;    // preds rows / columns per CTA
  int FYB, FXB;  // full-res rows / columns per footprint block
};

// first index dst in [0, out) whose tap (i1 when hi = false, i0 when hi = true) is >= i (hi = false) or > i (hi = true); out if none
__device__ int ce_first(int i, bool hi, float scale, int in, int out) {
  int lo = 0, up = out;
  while (lo < up) {
    const int mid = (lo + up) >> 1;
    int a, b;
    float l;
    bilinear_src(mid, scale, in, &a, &b, &l);
    const bool past = hi ? a > i : b >= i;
    if (past) up = mid;
    else lo = mid + 1;
  }
  return lo;
}

// weight of source index i in the taps (t0, t1, l1) of one output index
__device__ __forceinline__ float ce_weight(int i, int t0, int t1, float l1) { return (t0 == i ? 1.0f - l1 : 0.0f) + (t1 == i ? l1 : 0.0f); }

template <typename T>
__global__ void __launch_bounds__(kCeThreads) seg_ce_bwd_kernel(const float* __restrict__ x, const T* __restrict__ lab, CeShape S, CeTile K,
                                                                const float* __restrict__ lse, const long long* __restrict__ record,
                                                                const float* __restrict__ gout, float loss_weight, float* __restrict__ gx) {
  extern __shared__ float4 ce_smem[];
  const int bpx = K.FYB * K.FXB;
  float* G = reinterpret_cast<float*>(ce_smem);
  float* L = G + bpx;
  float* R = L + bpx;          // [FYB][TJ]
  float* rl = R + K.FYB * K.TJ;  // row weights l1 [FYB]
  float* cl = rl + K.FYB;        // column weights l1 [FXB]
  int* r0 = reinterpret_cast<int*>(cl + K.FXB);
  int* r1 = r0 + K.FYB;
  int* c0 = r1 + K.FYB;
  int* c1 = c0 + K.FXB;
  int* ylo = c1 + K.FXB;
  int* yhi = ylo + K.TI;
  int* xlo = yhi + K.TI;
  int* xhi = xlo + K.TJ;
  short* tg = reinterpret_cast<short*>(xhi + K.TJ);

  const int b = blockIdx.z, i0 = blockIdx.y * K.TI, j0 = blockIdx.x * K.TJ;
  const int ti = min(K.TI, S.h - i0), tj = min(K.TJ, S.w - j0), nout = ti * tj;
  const int hw = S.h * S.w;
  float* gb = gx + (size_t)b * S.C * hw + (size_t)i0 * S.w + j0;
  if (record[1] > 0) {  // a label outside [0, C): every gradient element is NaN
    for (int c = 0; c < S.C; ++c)
      for (int o = threadIdx.x; o < nout; o += kCeThreads) gb[(size_t)c * hw + (o / tj) * S.w + o % tj] = __int_as_float(0x7fffffff);
    return;
  }
  // every valid pixel carries g * loss_weight / n_valid; ignored pixels carry exactly 0 (also when n_valid = 0)
  const float s = (gout[0] * loss_weight) / (float)record[0];
  for (int t = threadIdx.x; t < ti + tj; t += kCeThreads) {
    if (t < ti) {
      ylo[t] = ce_first(i0 + t, false, S.scale_h, S.h, S.H);
      yhi[t] = ce_first(i0 + t, true, S.scale_h, S.h, S.H);
    } else {
      const int u = t - ti;
      xlo[u] = ce_first(j0 + u, false, S.scale_w, S.w, S.W);
      xhi[u] = ce_first(j0 + u, true, S.scale_w, S.w, S.W);
    }
  }
  __syncthreads();
  const int Y0 = ylo[0], Y1 = yhi[ti - 1], X0 = xlo[0], X1 = xhi[tj - 1];
  if (Y0 >= Y1 || X0 >= X1) {  // no full-res pixel reaches this tile (downsampling)
    for (int c = 0; c < S.C; ++c)
      for (int o = threadIdx.x; o < nout; o += kCeThreads) gb[(size_t)c * hw + (o / tj) * S.w + o % tj] = 0.0f;
    return;
  }
  const float* xb = x + (size_t)b * S.C * hw;
  const int ty = threadIdx.x >> 5, tx = threadIdx.x & 31;
  for (int by = Y0; by < Y1; by += K.FYB) {
    const int fy = min(K.FYB, Y1 - by);
    for (int bx = X0; bx < X1; bx += K.FXB) {
      const int fx = min(K.FXB, X1 - bx);
      const bool first = by == Y0 && bx == X0;
      for (int y = threadIdx.x; y < fy; y += kCeThreads) {
        int a, c;
        bilinear_src(by + y, S.scale_h, S.h, &a, &c, &rl[y]);
        r0[y] = a * S.w;
        r1[y] = c * S.w;
      }
      for (int u = threadIdx.x; u < fx; u += kCeThreads) bilinear_src(bx + u, S.scale_w, S.w, &c0[u], &c1[u], &cl[u]);
      for (int y = ty; y < fy; y += kCeThreads / 32) {
        for (int u = tx; u < fx; u += 32) {
          const int t = ce_target(lab, S, b, by + y, bx + u);
          tg[y * K.FXB + u] = (short)(t >= 0 ? t : kCeIgnore);  // (no label is out of range here: record[1] == 0)
          L[y * K.FXB + u] = lse[((size_t)b * S.H + by + y) * S.W + bx + u];
        }
      }
      __syncthreads();
      for (int c = 0; c < S.C; ++c) {
        const float* xc = xb + (size_t)c * hw;
        // G = s (softmax - onehot) over the block
        for (int y = ty; y < fy; y += kCeThreads / 32) {
          const int a0 = r0[y], a1 = r1[y];
          const float lh1 = rl[y], lh0 = 1.0f - lh1;
#pragma unroll 4
          for (int u = tx; u < fx; u += 32) {
            const int k = y * K.FXB + u;
            const int t = tg[k];
            const float lw1 = cl[u];
            float g = 0.0f;
            if (t >= 0) {
              const float z = ce_interp(xc, a0, a1, c0[u], c1[u], lh0, lh1, 1.0f - lw1, lw1);
              g = s * (expf(z - L[k]) - (c == t ? 1.0f : 0.0f));
            }
            G[k] = g;
          }
        }
        __syncthreads();
        // along each footprint row into the tile's columns
        for (int o = threadIdx.x; o < fy * tj; o += kCeThreads) {
          const int y = o / tj, u = o - y * tj, j = j0 + u;
          const int xa = max(xlo[u], bx) - bx, xe = min(xhi[u], bx + fx) - bx;
          float acc = 0.0f;
          for (int q = xa; q < xe; ++q) acc += ce_weight(j, c0[q], c1[q], cl[q]) * G[y * K.FXB + q];
          R[y * K.TJ + u] = acc;
        }
        __syncthreads();
        // along the footprint columns into the tile's rows
        for (int o = threadIdx.x; o < nout; o += kCeThreads) {
          const int v = o / tj, u = o - v * tj, i = i0 + v;
          const int ya = max(ylo[v], by) - by, ye = min(yhi[v], by + fy) - by;
          float acc = 0.0f;
          for (int q = ya; q < ye; ++q) acc += ce_weight(i * S.w, r0[q], r1[q], rl[q]) * R[q * K.TJ + u];
          float* d = gb + (size_t)c * hw + v * S.w + u;
          *d = first ? acc : *d + acc;
        }
      }
      __syncthreads();  // the next block restages the taps, labels and lse
    }
  }
}

// --------------------------------------------------------------------------------------------------------------------------- host
inline int fwd_blocks(long long n) { return (int)((n + (long long)kCeThreads * kCePix - 1) / ((long long)kCeThreads * kCePix)); }

inline size_t ws_bytes_for(long long n) { return align_up((size_t)fwd_blocks(n) * 3 * sizeof(double), 256); }

inline int pow2_at_most(double v, int hi) {
  int p = 1;
  while (p * 2 <= hi && p * 2 <= v) p *= 2;
  return p;
}

// Tile of about 32 x 128 full-res pixels; blocks as large as the footprint up to kCeBlockPix pixels (a larger footprint takes several).
CeTile ce_tile(const CeShape& S) {
  CeTile K;
  K.TI = pow2_at_most(32.0 * S.h / S.H, kCeMaxTI);
  K.TJ = pow2_at_most(128.0 * S.w / S.W, kCeMaxTJ);
  // (a footprint spans the tile's full-res rows plus up to two on each side: 36 x 132 for the 8 x 32 tile at x4)
  const long long fy = (long long)ceil((double)K.TI * S.H / S.h) + 4, fx = (long long)ceil((double)K.TJ * S.W / S.w) + 4;
  K.FXB = (int)(fx < 1024 ? fx : 1024);
  long long fyb = fy;
  if (fyb > kCeBlockPix / K.FXB) fyb = kCeBlockPix / K.FXB;
  if (fyb > kCeBlockPix / K.TJ) fyb = kCeBlockPix / K.TJ;
  K.FYB = (int)(fyb < 1 ? 1 : fyb);
  return K;
}

size_t ce_smem_bytes(const CeTile& K) {
  const size_t bpx = (size_t)K.FYB * K.FXB;
  return (2 * bpx + (size_t)K.FYB * K.TJ + K.FYB + K.FXB) * 4 + (2 * (size_t)K.FYB + 2 * K.FXB + 2 * K.TI + 2 * K.TJ) * 4 + bpx * 2;
}

// Validates what the forward and the backward share and fills S.
int make_shape(const char* what, const float* preds, int32_t B, int32_t C, int32_t h, int32_t w, const void* labels, int32_t dtype, int32_t H,
               int32_t W, int64_t sb, int64_t sh, int64_t sw, int64_t ignore_index, CeShape* S) {
  CVB_REQUIRE(C >= 1 && C <= kCeNcMax, "%s: C must be in [1, %d] (got %d)", what, kCeNcMax, C);
  CVB_REQUIRE(B >= 1 && B <= kCeMaxDim, "%s: B must be in [1, %d] (got %d)", what, kCeMaxDim, B);
  CVB_REQUIRE(h >= 1 && w >= 1 && h <= kCeMaxDim && w <= kCeMaxDim, "%s: preds h, w must be in [1, %d] (got %d x %d)", what, kCeMaxDim, h, w);
  CVB_REQUIRE(H >= 1 && W >= 1 && H <= kCeMaxDim && W <= kCeMaxDim, "%s: label H, W must be in [1, %d] (got %d x %d)", what, kCeMaxDim, H, W);
  CVB_REQUIRE((long long)B * H * W <= INT_MAX, "%s: B x H x W must be below 2^31 (got %lld)", what, (long long)B * H * W);
  CVB_REQUIRE((long long)h * w <= INT_MAX, "%s: h x w must be below 2^31", what);
  CVB_REQUIRE(dtype == CVB_SEG_U8 || dtype == CVB_SEG_I32 || dtype == CVB_SEG_I64, "%s: unknown label dtype code %d", what, dtype);
  CVB_REQUIRE(sb >= 0 && sh >= 0 && sw >= 0, "%s: label strides must be >= 0 (got %lld, %lld, %lld)", what, (long long)sb, (long long)sh,
              (long long)sw);
  CVB_REQUIRE((B - 1) * sb + (H - 1) * sh + (W - 1) * sw < (1LL << 40), "%s: label strides too large", what);
  CVB_REQUIRE(preds && is_aligned(preds, 4), "%s: preds missing or not 4-byte aligned", what);
  CVB_REQUIRE(labels && is_aligned(labels, seg_label_bytes(dtype)), "%s: labels missing or not aligned to their element size", what);
  *S = CeShape{B, C, h, w, H, W, sb, sh, sw, ignore_index, (float)h / (float)H, (float)w / (float)W};
  return CVB_OK;
}

}  // namespace
}  // namespace cvb

using namespace cvb;

extern "C" int32_t cvb_train_seg_ce_nc_max(void) { return kCeNcMax; }

extern "C" size_t cvb_train_seg_ce_workspace_bytes(int32_t B, int32_t H, int32_t W) {
  if (B <= 0 || H <= 0 || W <= 0 || (long long)B * H * W > INT_MAX) return 0;
  return ws_bytes_for((long long)B * H * W);
}

extern "C" int cvb_train_seg_ce_fwd(const float* preds, int32_t B, int32_t C, int32_t h, int32_t w, const void* labels, int32_t label_dtype,
                                    int32_t H, int32_t W, int64_t sb, int64_t sh, int64_t sw, int64_t ignore_index, float loss_weight,
                                    float* lse, int64_t* record, float* loss, void* workspace, size_t ws_bytes, void* stream) {
  CeShape S;
  const int rc = make_shape("train_seg_ce_fwd", preds, B, C, h, w, labels, label_dtype, H, W, sb, sh, sw, ignore_index, &S);
  if (rc != CVB_OK) return rc;
  CVB_REQUIRE(lse && record && loss && is_aligned(lse, 4) && is_aligned(record, 8) && is_aligned(loss, 4),
              "train_seg_ce_fwd: lse, loss (4-byte aligned) and record (8-byte aligned) are required");
  const long long n = (long long)B * H * W;
  CVB_REQUIRE(workspace && is_aligned(workspace, 256), "train_seg_ce_fwd: workspace required, 256-byte aligned");
  CVB_REQUIRE(ws_bytes >= ws_bytes_for(n), "train_seg_ce_fwd: workspace of %zu bytes too small (%zu needed)", ws_bytes, ws_bytes_for(n));
  double* partial = static_cast<double*>(workspace);
  const int nblk = fwd_blocks(n);
  cudaStream_t st = as_stream(stream);
  switch (label_dtype) {
    case CVB_SEG_U8: seg_ce_fwd_kernel<<<nblk, kCeThreads, 0, st>>>(preds, static_cast<const uint8_t*>(labels), S, lse, partial); break;
    case CVB_SEG_I32: seg_ce_fwd_kernel<<<nblk, kCeThreads, 0, st>>>(preds, static_cast<const int32_t*>(labels), S, lse, partial); break;
    default: seg_ce_fwd_kernel<<<nblk, kCeThreads, 0, st>>>(preds, static_cast<const long long*>(labels), S, lse, partial); break;
  }
  seg_ce_final_kernel<<<1, kCeFinalThreads, 0, st>>>(partial, nblk, loss_weight, loss, reinterpret_cast<long long*>(record));
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch(2);
  return CVB_OK;
}

template <typename T>
static int ce_bwd_launch(const float* preds, const T* labels, const CeShape& S, const float* lse, const int64_t* record, const float* grad_out,
                         float loss_weight, float* grad_preds, cudaStream_t st) {
  const CeTile K = ce_tile(S);
  const size_t smem = ce_smem_bytes(K);
  auto fn = seg_ce_bwd_kernel<T>;
  CVB_CHECK_CUDA(opt_in_smem(fn, (int)smem));
  const dim3 grid(ceil_div(S.w, K.TJ), ceil_div(S.h, K.TI), S.B);
  fn<<<grid, kCeThreads, smem, st>>>(preds, labels, S, K, lse, reinterpret_cast<const long long*>(record), grad_out, loss_weight, grad_preds);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}

extern "C" int cvb_train_seg_ce_bwd(const float* preds, int32_t B, int32_t C, int32_t h, int32_t w, const void* labels, int32_t label_dtype,
                                    int32_t H, int32_t W, int64_t sb, int64_t sh, int64_t sw, int64_t ignore_index, float loss_weight,
                                    const float* lse, const int64_t* record, const float* grad_out, float* grad_preds, void* stream) {
  CeShape S;
  const int rc = make_shape("train_seg_ce_bwd", preds, B, C, h, w, labels, label_dtype, H, W, sb, sh, sw, ignore_index, &S);
  if (rc != CVB_OK) return rc;
  CVB_REQUIRE(lse && record && grad_out && grad_preds && is_aligned(lse, 4) && is_aligned(record, 8) && is_aligned(grad_out, 4) && is_aligned(grad_preds, 4),
              "train_seg_ce_bwd: lse, grad_out, grad_preds (4-byte aligned) and record (8-byte aligned) are required");
  const cudaStream_t st = as_stream(stream);
  switch (label_dtype) {
    case CVB_SEG_U8: return ce_bwd_launch(preds, static_cast<const uint8_t*>(labels), S, lse, record, grad_out, loss_weight, grad_preds, st);
    case CVB_SEG_I32: return ce_bwd_launch(preds, static_cast<const int32_t*>(labels), S, lse, record, grad_out, loss_weight, grad_preds, st);
    default: return ce_bwd_launch(preds, static_cast<const long long*>(labels), S, lse, record, grad_out, loss_weight, grad_preds, st);
  }
}
