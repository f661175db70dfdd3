// The YOLOv6 training loss on the device: target packing, the ATSS and task-aligned (TAL) assigners, the GIoU / SIoU box loss and its
// gradient with respect to pred_distri (src/losses/det/yolov6_loss.py with src/models/assigners/; the algorithm is restated in
// oracle/yolov6_loss_oracle.py).
//
// Forward (cvb_train_yolov6_loss_fwd), all stream-ordered, no host sync, CUDA-graph capturable:
//   1. v6_pack_kernel     one CTA per image: the image's GT rows of gt [nt, 6] in input order (fp64 scale and xywh -> xyxy), its slot
//                         range, and zeroed per-anchor claim counters.
//   2. v6_select_kernel   one warp per GT slot: ATSS (the min(9, level size) nearest anchors per level, threshold mean + unbiased std of
//                         their IoUs) or TAL (the 13 largest score^1 IoU^6 metrics); every positive (GT, anchor) pair claims its anchor
//                         with integer atomics (a count and the lowest claiming slot).
//   3. v6_resolve_kernel  one thread per (image, anchor): the anchor's GT (a single claimant, or the first IoU maximum over all of the
//                         image's rows when several claim it), its targets, and (TAL) the per-GT maxima of the alignment metric and IoU as
//                         integer atomic maxima of order-preserving keys.
//   4. v6_loss_kernel     one thread per (image, anchor): the soft label (TAL: align pos_iou / (pos_align + 1e-9)) and weight (1 - IoU)
//                         terms, summed per CTA in fp64.
//   5. v6_final_kernel    one CTA: the CTA partials in a fixed order -> stats and the three outputs.
// Backward (cvb_train_yolov6_loss_bwd): v6_bwd_kernel writes every element of the pred_distri gradient from the saved assignment.
// Nothing of size [B, n_max_boxes, A] exists: the largest buffers are per anchor.  No float atomics: results are bitwise reproducible.
//
// Ties: topk's order on equal values is not defined by torch; the kernels take the lowest anchor index among equal distances (ATSS) or
// equal metrics (TAL).  Precision: the assignment runs in the reference's fp64 / fp32 operation order (this file is compiled with
// --fmad=false); the box loss and its gradient in fp64, the gradient along autograd's rules at the kinks (torch.min / max split a tie,
// clamp(0) passes at the bound, abs'(0) = 0, SIoU's where routes to its selected branch).
#include <limits.h>

#include "internal.h"

namespace cvb {
namespace {

constexpr int kV6Threads = 256;
constexpr int kV6SelWarps = 4;           // warps (GT slots) per select CTA
constexpr int kV6AtssK = 9;              // ATSS candidates per level
constexpr int kV6TalK = 13;              // TAL top-k
constexpr int kV6MaxCand = kV6AtssK * CVB_YOLOV6_MAX_LEVELS;
constexpr int kV6FinalThreads = 256;

struct V6Levels {
  int nlev, A, B, nc, nt, mode, siou;
  int off[CVB_YOLOV6_MAX_LEVELS + 1];
  int w[CVB_YOLOV6_MAX_LEVELS];
  float stride[CVB_YOLOV6_MAX_LEVELS];
  float half[CVB_YOLOV6_MAX_LEVELS];     // grid_cell_size * stride * 0.5, as fp32
  float offset, scale;                    // grid_cell_offset; ori_img_size
  double wt[3];                           // loss weights of the (iou, dfl, class) outputs
  int nblk;
};

struct Anchor {
  float sx, sy;    // anchor point (pixels): (column + offset) * stride
  float ax1, ay1, ax2, ay2;  // ATSS anchor box: point -+ grid_cell_size * stride / 2
  float s;         // stride
};

__device__ __forceinline__ Anchor anchor_at(const V6Levels& L, int a) {
  int l = 0;
#pragma unroll
  for (int k = 1; k < CVB_YOLOV6_MAX_LEVELS; ++k)
    if (k < L.nlev && a >= L.off[k]) l = k;
  const int i = a - L.off[l];
  Anchor r;
  r.s = L.stride[l];
  r.sx = __fmul_rn(__fadd_rn((float)(i % L.w[l]), L.offset), r.s);
  r.sy = __fmul_rn(__fadd_rn((float)(i / L.w[l]), L.offset), r.s);
  r.ax1 = __fsub_rn(r.sx, L.half[l]);
  r.ay1 = __fsub_rn(r.sy, L.half[l]);
  r.ax2 = __fadd_rn(r.sx, L.half[l]);
  r.ay2 = __fadd_rn(r.sy, L.half[l]);
  return r;
}

// pred box in stride units (dist2bbox of pred_distri about anchor_points / stride), fp32
__device__ __forceinline__ float4 pred_box(const float* __restrict__ distri, size_t ba, const Anchor& an) {
  const float4 d = reinterpret_cast<const float4*>(distri)[ba];
  const float px = __fdiv_rn(an.sx, an.s), py = __fdiv_rn(an.sy, an.s);
  return make_float4(__fsub_rn(px, d.x), __fsub_rn(py, d.y), __fadd_rn(px, d.z), __fadd_rn(py, d.w));
}
__device__ __forceinline__ float4 times(float4 b, float s) {
  return make_float4(__fmul_rn(b.x, s), __fmul_rn(b.y, s), __fmul_rn(b.z, s), __fmul_rn(b.w, s));
}

__device__ __forceinline__ double dmax0(double x) { return x < 0.0 ? 0.0 : x; }

// iou_calculator (assigner_utils): GT fp64 against an fp32 box, areas clipped at 0, eps 1e-9; the fp32 box's area is fp32
__device__ __forceinline__ double iou_calc(double4 g, float4 p) {
  const double ow = dmax0(fmin(g.z, (double)p.z) - fmax(g.x, (double)p.x)), oh = dmax0(fmin(g.w, (double)p.w) - fmax(g.y, (double)p.y));
  const double ov = ow * oh;
  const double a1 = dmax0(g.z - g.x) * dmax0(g.w - g.y);
  const float pw = __fsub_rn(p.z, p.x), ph = __fsub_rn(p.w, p.y);
  const float a2 = __fmul_rn(pw < 0.0f ? 0.0f : pw, ph < 0.0f ? 0.0f : ph);
  return ov / (((a1 + (double)a2) - ov) + 1e-9);
}

// bbox_overlaps (mode 'iou', not aligned) of a GT against an ATSS anchor box: union clamped to 1e-6
__device__ __forceinline__ double iou_anchor(double4 g, const Anchor& an) {
  const double a1 = (g.z - g.x) * (g.w - g.y);
  const float a2 = __fmul_rn(__fsub_rn(an.ax2, an.ax1), __fsub_rn(an.ay2, an.ay1));
  const double ow = dmax0(fmin(g.z, (double)an.ax2) - fmax(g.x, (double)an.ax1));
  const double oh = dmax0(fmin(g.w, (double)an.ay2) - fmax(g.y, (double)an.ay1));
  const double ov = ow * oh;
  return ov / fmax((a1 + (double)a2) - ov, 1e-6);
}

// select_candidates_in_gts: the anchor point strictly inside the GT, min delta > 1e-9
__device__ __forceinline__ bool in_gt(double4 g, float x, float y) {
  const double X = x, Y = y;
  return fmin(fmin(X - g.x, Y - g.y), fmin(g.z - X, g.w - Y)) > 1e-9;
}

// Order-preserving uint64 key of a double (atomicMax of keys = max of values)
__device__ __forceinline__ unsigned long long dkey(double v) {
  const unsigned long long u = (unsigned long long)__double_as_longlong(v);
  return (u >> 63) ? ~u : (u | 0x8000000000000000ULL);
}
__device__ __forceinline__ double dkey_value(unsigned long long k) {
  return __longlong_as_double((long long)((k >> 63) ? (k & 0x7FFFFFFFFFFFFFFFULL) : ~k));
}

// ------------------------------------------------------------------------------------------------------------------ box loss
// A value with its derivatives with respect to pred_distri's (l, t, r, b): the forward takes v, the backward d.  One formula serves both.
struct D {
  double v, d[4];
};
__device__ __forceinline__ D dc(double v) { return D{v, {0.0, 0.0, 0.0, 0.0}}; }
__device__ __forceinline__ D scale(const D& a, double v, double k) {
  D r{v, {}};
#pragma unroll
  for (int i = 0; i < 4; ++i) r.d[i] = a.d[i] * k;
  return r;
}
__device__ __forceinline__ D operator+(const D& a, const D& b) {
  D r{a.v + b.v, {}};
#pragma unroll
  for (int i = 0; i < 4; ++i) r.d[i] = a.d[i] + b.d[i];
  return r;
}
__device__ __forceinline__ D operator-(const D& a, const D& b) {
  D r{a.v - b.v, {}};
#pragma unroll
  for (int i = 0; i < 4; ++i) r.d[i] = a.d[i] - b.d[i];
  return r;
}
__device__ __forceinline__ D operator+(const D& a, double b) { return D{a.v + b, {a.d[0], a.d[1], a.d[2], a.d[3]}}; }
__device__ __forceinline__ D operator-(double a, const D& b) { return scale(b, a - b.v, -1.0); }
__device__ __forceinline__ D operator*(const D& a, const D& b) {
  D r{a.v * b.v, {}};
#pragma unroll
  for (int i = 0; i < 4; ++i) r.d[i] = a.d[i] * b.v + b.d[i] * a.v;
  return r;
}
__device__ __forceinline__ D operator*(const D& a, double k) { return scale(a, a.v * k, k); }
__device__ __forceinline__ D operator/(const D& a, const D& b) {
  D r{a.v / b.v, {}};
#pragma unroll
  for (int i = 0; i < 4; ++i) r.d[i] = (a.d[i] - r.v * b.d[i]) / b.v;
  return r;
}
// the value rounded to fp32 (an fp32 tensor op of the reference), the derivative that of the exact operation
__device__ __forceinline__ D r32(D a) {
  a.v = (double)(float)a.v;
  return a;
}
// torch.minimum / maximum: the gradient goes to the smaller / larger input, half to each on a tie
__device__ __forceinline__ D tmin(const D& a, const D& b) {
  if (a.v < b.v) return a;
  if (b.v < a.v) return b;
  D r{a.v, {}};
#pragma unroll
  for (int i = 0; i < 4; ++i) r.d[i] = 0.5 * (a.d[i] + b.d[i]);
  return r;
}
__device__ __forceinline__ D tmax(const D& a, const D& b) {
  if (a.v > b.v) return a;
  if (b.v > a.v) return b;
  D r{a.v, {}};
#pragma unroll
  for (int i = 0; i < 4; ++i) r.d[i] = 0.5 * (a.d[i] + b.d[i]);
  return r;
}
__device__ __forceinline__ D clamp0(const D& a) { return a.v >= 0.0 ? a : dc(0.0); }
__device__ __forceinline__ D dabs(const D& a) { return scale(a, fabs(a.v), a.v > 0.0 ? 1.0 : (a.v < 0.0 ? -1.0 : 0.0)); }
__device__ __forceinline__ D dsqrt(const D& a) { return scale(a, sqrt(a.v), 0.5 * pow(a.v, -0.5)); }
__device__ __forceinline__ D dexp(const D& a) {
  const double e = exp(a.v);
  return scale(a, e, e);
}
__device__ __forceinline__ D dpow4(const D& a) { return scale(a, pow(a.v, 4.0), 4.0 * pow(a.v, 3.0)); }
__device__ __forceinline__ D dasin(const D& a) { return scale(a, asin(a.v), 1.0 / sqrt(1.0 - a.v * a.v)); }
__device__ __forceinline__ D dcos(const D& a) { return scale(a, cos(a.v), -sin(a.v)); }

// 1 - GIoU / 1 - SIoU (IOUloss, xyxy, eps 1e-10) of the fp32 pred box (stride units, from pred_distri d about the anchor point (px, py))
// against the fp64 target box (stride units).  w1, h1 and w1 h1 are fp32 in the reference.
__device__ D box_loss(float4 d, float px, float py, double4 t, bool siou) {
  const double eps = 1e-10;
  const D x1{(double)__fsub_rn(px, d.x), {-1.0, 0.0, 0.0, 0.0}}, y1{(double)__fsub_rn(py, d.y), {0.0, -1.0, 0.0, 0.0}};
  const D x2{(double)__fadd_rn(px, d.z), {0.0, 0.0, 1.0, 0.0}}, y2{(double)__fadd_rn(py, d.w), {0.0, 0.0, 0.0, 1.0}};
  const D tx1 = dc(t.x), ty1 = dc(t.y), tx2 = dc(t.z), ty2 = dc(t.w);
  const D inter = clamp0(tmin(x2, tx2) - tmax(x1, tx1)) * clamp0(tmin(y2, ty2) - tmax(y1, ty1));
  const D w1 = r32(x2 - x1), h1 = r32(r32(y2 - y1) + (double)1e-10f);
  const double w2 = t.z - t.x, h2 = (t.w - t.y) + eps;
  const D uni = ((r32(w1 * h1) + w2 * h2) - inter) + eps;
  const D iou = inter / uni;
  const D cw = tmax(x2, tx2) - tmin(x1, tx1), ch = tmax(y2, ty2) - tmin(y1, ty1);
  if (!siou) {
    const D c = cw * ch + eps;
    return 1.0 - (iou - (c - uni) / c);
  }
  const D scw = ((dc(t.x + t.z) - x1) - x2) * 0.5 + eps, sch = ((dc(t.y + t.w) - y1) - y2) * 0.5 + eps;
  const D sigma = dsqrt(scw * scw + sch * sch);
  const D s1 = dabs(scw) / sigma, s2 = dabs(sch) / sigma;
  const D sa = s1.v > 0.7071067811865476 ? s2 : s1;
  const D angle = dcos(dasin(sa) * 2.0 + (-1.5707963267948966));
  const D rx = (scw / cw) * (scw / cw), ry = (sch / ch) * (sch / ch);
  const D gamma = angle + (-2.0);
  const D dist = (2.0 - dexp(gamma * rx)) - dexp(gamma * ry);
  const D W2 = dc(w2), H2 = dc(h2);
  const D ow = dabs(w1 - W2) / tmax(w1, W2), oh = dabs(h1 - H2) / tmax(h1, H2);
  const D shape = dpow4(1.0 - dexp(ow * -1.0)) + dpow4(1.0 - dexp(oh * -1.0));
  return 1.0 - (iou - (dist + shape) * 0.5);
}

// ------------------------------------------------------------------------------------------------------------------ forward
struct V6Ws {
  int32_t *img_start, *img_count;   // [B]
  double4* gbox;                     // [nt] xyxy pixels, slot order
  int32_t *glab, *gimg;              // [nt] truncated label (INT_MIN if out of int range), image
  uint8_t* gmask;                    // [nt] mask_gt
  unsigned long long *pos_align, *pos_iou;  // [nt] TAL per-GT maxima (keys)
  int32_t *claims, *claimant;        // [B, A]
  double *align, *iou;               // [B, A] TAL metric and IoU of the anchor's GT
  double* partial;                   // [B nblk, 4]
  size_t bytes;
};

V6Ws v6_ws(void* base, int B, int A, int nt, int nblk) {
  WsCarver c(base);
  V6Ws w{};
  const size_t n = (size_t)(nt > 0 ? nt : 1), ba = (size_t)B * A;
  w.img_start = static_cast<int32_t*>(c.take((size_t)B * 4));
  w.img_count = static_cast<int32_t*>(c.take((size_t)B * 4));
  w.gbox = static_cast<double4*>(c.take(n * sizeof(double4)));
  w.glab = static_cast<int32_t*>(c.take(n * 4));
  w.gimg = static_cast<int32_t*>(c.take(n * 4));
  w.gmask = static_cast<uint8_t*>(c.take(n));
  w.pos_align = static_cast<unsigned long long*>(c.take(n * 8));
  w.pos_iou = static_cast<unsigned long long*>(c.take(n * 8));
  w.claims = static_cast<int32_t*>(c.take(ba * 4));
  w.claimant = static_cast<int32_t*>(c.take(ba * 4));
  w.align = static_cast<double*>(c.take(ba * 8));
  w.iou = static_cast<double*>(c.take(ba * 8));
  w.partial = static_cast<double*>(c.take((size_t)B * nblk * 4 * sizeof(double)));
  w.bytes = c.bytes();
  return w;
}

// image index of a row: int() truncation, rows outside [0, B) dropped (-1)
__device__ __forceinline__ int row_image(double v, int B) { return (v > -1.0 && v < (double)B) ? (int)v : -1; }

__global__ void __launch_bounds__(kV6Threads) v6_pack_kernel(V6Levels L, const double* __restrict__ gt, V6Ws w) {
  __shared__ int wsum[2][kV6Threads / 32];
  const int b = blockIdx.x, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int a = threadIdx.x; a < L.A; a += blockDim.x) {
    w.claims[(size_t)b * L.A + a] = 0;
    w.claimant[(size_t)b * L.A + a] = INT_MAX;
  }
  // rows before this image's first slot: every in-range row of a lower image
  int before = 0, mine = 0;
  for (int r = threadIdx.x; r < L.nt; r += blockDim.x) {
    const int im = row_image(gt[(size_t)r * 6], L.B);
    before += (im >= 0 && im < b);
  }
  for (int o = 16; o; o >>= 1) before += __shfl_xor_sync(0xffffffffu, before, o);
  if (lane == 0) wsum[0][wid] = before;
  __syncthreads();
  int start = 0;
  for (int k = 0; k < kV6Threads / 32; ++k) start += wsum[0][k];
  // this image's rows in input order: chunks of blockDim rows, ranked by a block scan of the match flags
  int base = start;
  for (int r0 = 0; r0 < L.nt; r0 += blockDim.x) {
    const int r = r0 + threadIdx.x;
    const bool hit = r < L.nt && row_image(gt[(size_t)r * 6], L.B) == b;
    const unsigned m = __ballot_sync(0xffffffffu, hit);
    __syncthreads();
    if (lane == 0) wsum[1][wid] = __popc(m);
    __syncthreads();
    int pre = 0, tot = 0;
    for (int k = 0; k < kV6Threads / 32; ++k) {
      pre += k < wid ? wsum[1][k] : 0;
      tot += wsum[1][k];
    }
    if (hit) {
      const int s = base + pre + __popc(m & ((1u << lane) - 1u));
      const double* row = gt + (size_t)r * 6;
      // preprocess: (cx, cy, w, h) * ori_img_size in fp64, then x1 = cx - w 0.5, y1 = cy - h 0.5, x2 = x1 + w, y2 = y1 + h
      const double sc = (double)L.scale;
      const double cx = row[2] * sc, cy = row[3] * sc, bw = row[4] * sc, bh = row[5] * sc;
      const double x1 = cx - bw * 0.5, y1 = cy - bh * 0.5;
      const double4 g = make_double4(x1, y1, x1 + bw, y1 + bh);
      w.gbox[s] = g;
      const double lab = row[1];
      w.glab[s] = (lab > -2147483648.0 && lab < 2147483648.0) ? (int)lab : INT_MIN;
      w.gimg[s] = b;
      w.gmask[s] = (((g.x + g.y) + g.z) + g.w) > 0.0;
      w.pos_align[s] = dkey(0.0);  // the maxima include the zeros of the anchors that are not the GT's positives
      w.pos_iou[s] = dkey(0.0);
    }
    base += tot;
    mine += tot;
  }
  if (threadIdx.x == 0) {
    w.img_start[b] = start;
    w.img_count[b] = mine;
  }
}

// Candidate order: ATSS ascending distance, TAL descending metric; the lower anchor index first on equal values.
template <bool kLargest>
__device__ __forceinline__ bool before_(double v, int i, double u, int j) {
  return kLargest ? (v > u || (v == u && i < j)) : (v < u || (v == u && i < j));
}

// A lane's K best (value, anchor) pairs, kept sorted in registers (fully unrolled: no local memory).
template <int K, bool kLargest>
struct TopK {
  double v[K];
  int i[K];
  __device__ __forceinline__ void init() {
#pragma unroll
    for (int k = 0; k < K; ++k) {
      v[k] = kLargest ? -INFINITY : INFINITY;
      i[k] = INT_MAX;
    }
  }
  __device__ __forceinline__ void push(double x, int a) {
    if (!before_<kLargest>(x, a, v[K - 1], i[K - 1])) return;
    v[K - 1] = x;
    i[K - 1] = a;
#pragma unroll
    for (int k = K - 1; k > 0; --k) {
      if (before_<kLargest>(v[k], i[k], v[k - 1], i[k - 1])) {
        const double tv = v[k];
        v[k] = v[k - 1];
        v[k - 1] = tv;
        const int ti = i[k];
        i[k] = i[k - 1];
        i[k - 1] = ti;
      }
    }
  }
  // Warp-wide: the first n (<= K) pairs of the merged lists; lane r < n gets the r-th anchor index (INT_MAX: none).
  __device__ __forceinline__ int merge(int n, int lane) {
    int mine = INT_MAX;
    for (int r = 0; r < n; ++r) {
      double bv = v[0];
      int bi = i[0];
#pragma unroll
      for (int o = 16; o; o >>= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (before_<kLargest>(ov, oi, bv, bi)) {
          bv = ov;
          bi = oi;
        }
      }
      if (lane == r) mine = bi;
      if (bi != INT_MAX && i[0] == bi) {  // the owner pops its head
#pragma unroll
        for (int k = 0; k < K - 1; ++k) {
          v[k] = v[k + 1];
          i[k] = i[k + 1];
        }
        v[K - 1] = kLargest ? -INFINITY : INFINITY;
        i[K - 1] = INT_MAX;
      }
    }
    return mine;
  }
};

__device__ __forceinline__ void claim(const V6Ws& w, int A, int b, int a, int slot) {
  atomicAdd(&w.claims[(size_t)b * A + a], 1);
  atomicMin(&w.claimant[(size_t)b * A + a], slot);
}

__global__ void __launch_bounds__(kV6SelWarps * 32) v6_atss_select_kernel(V6Levels L, V6Ws w) {
  __shared__ int s_idx[kV6SelWarps][kV6MaxCand];
  __shared__ double s_iou[kV6SelWarps][kV6MaxCand];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int slot = blockIdx.x * kV6SelWarps + wid;
  // slots past the packed rows (dropped rows) and mask_gt = 0 GTs select nothing
  if (slot >= L.nt || slot >= w.img_start[L.B - 1] + w.img_count[L.B - 1] || !w.gmask[slot]) return;
  const int b = w.gimg[slot];
  const double4 g = w.gbox[slot];
  const double gcx = (g.x + g.z) / 2.0, gcy = (g.y + g.w) / 2.0;
  int n = 0;
  for (int l = 0; l < L.nlev; ++l) {
    TopK<kV6AtssK, false> top;
    top.init();
    for (int a = L.off[l] + lane; a < L.off[l + 1]; a += 32) {
      const Anchor an = anchor_at(L, a);
      const float acx = __fdiv_rn(__fadd_rn(an.ax1, an.ax2), 2.0f), acy = __fdiv_rn(__fadd_rn(an.ay1, an.ay2), 2.0f);
      const double dx = gcx - (double)acx, dy = gcy - (double)acy;
      top.push(sqrt(dx * dx + dy * dy), a);
    }
    const int k = min(kV6AtssK, L.off[l + 1] - L.off[l]);
    const int a = top.merge(k, lane);
    if (lane < k) {
      s_idx[wid][n + lane] = a;
      s_iou[wid][n + lane] = iou_anchor(g, anchor_at(L, a));
    }
    n += k;
  }
  __syncwarp();
  // threshold: mean + unbiased std of the candidates' IoUs, summed in candidate order
  double sum = 0.0;
  for (int k = 0; k < n; ++k) sum += s_iou[wid][k];
  const double mean = sum / (double)n;
  double ss = 0.0;
  for (int k = 0; k < n; ++k) {
    const double e = s_iou[wid][k] - mean;
    ss += e * e;
  }
  const double thr = mean + sqrt(ss / (double)(n - 1));
  for (int k = lane; k < n; k += 32) {
    const int a = s_idx[wid][k];
    const Anchor an = anchor_at(L, a);
    const float acx = __fdiv_rn(__fadd_rn(an.ax1, an.ax2), 2.0f), acy = __fdiv_rn(__fadd_rn(an.ay1, an.ay2), 2.0f);
    if (s_iou[wid][k] > thr && in_gt(g, acx, acy)) claim(w, L.A, b, a, slot);
  }
}

// class score of a label (0 outside [0, nc))
__device__ __forceinline__ float class_score(const V6Levels& L, const float* __restrict__ scores, size_t ba, int lab) {
  return (lab >= 0 && lab < L.nc) ? scores[ba * L.nc + lab] : 0.0f;
}

// TAL alignment metric: score^1 * IoU(GT, pred box)^6 in fp64
__device__ __forceinline__ double tal_metric(float sc, double iou) { return (double)sc * pow(iou, 6.0); }

__global__ void __launch_bounds__(kV6SelWarps * 32) v6_tal_select_kernel(V6Levels L, const float* __restrict__ scores, const float* __restrict__ distri,
                                                                         V6Ws w) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int slot = blockIdx.x * kV6SelWarps + wid;
  if (slot >= L.nt || slot >= w.img_start[L.B - 1] + w.img_count[L.B - 1] || !w.gmask[slot]) return;
  const int b = w.gimg[slot];
  const double4 g = w.gbox[slot];
  const int lab = w.glab[slot];
  TopK<kV6TalK, true> top;
  top.init();
  for (int a = lane; a < L.A; a += 32) {
    const Anchor an = anchor_at(L, a);
    double m = 0.0;
    if (in_gt(g, an.sx, an.sy)) {
      const size_t ba = (size_t)b * L.A + a;
      m = tal_metric(class_score(L, scores, ba, lab), iou_calc(g, times(pred_box(distri, ba, an), an.s)));
    }
    top.push(m, a);
  }
  const int a = top.merge(kV6TalK, lane);
  if (lane < kV6TalK && a != INT_MAX) {
    const Anchor an = anchor_at(L, a);
    if (in_gt(g, an.sx, an.sy)) claim(w, L.A, b, a, slot);
  }
}

__global__ void __launch_bounds__(kV6Threads) v6_resolve_kernel(V6Levels L, const float* __restrict__ scores, const float* __restrict__ distri, V6Ws w,
                                                                uint8_t* __restrict__ fg, int32_t* __restrict__ gt_idx, int32_t* __restrict__ labels,
                                                                double* __restrict__ tbox) {
  const int b = blockIdx.y, a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= L.A) return;
  const size_t ba = (size_t)b * L.A + a;
  const int start = w.img_start[b], cnt = w.img_count[b];
  const Anchor an = anchor_at(L, a);
  const float4 pd = times(pred_box(distri, ba, an), an.s);
  const int nclaim = w.claims[ba];
  int s = -1;
  if (nclaim == 1) {
    s = w.claimant[ba];
  } else if (nclaim > 1) {  // the first IoU maximum over all of the image's rows (padding rows have IoU 0 and come last)
    double best = 0.0;
    for (int k = 0; k < cnt; ++k) {
      const double4 g = w.gbox[start + k];
      const double v = L.mode == CVB_YOLOV6_ATSS ? iou_anchor(g, an) : iou_calc(g, pd);
      if (k == 0 || v > best) {
        best = v;
        s = start + k;
      }
    }
  }
  fg[ba] = s >= 0;
  gt_idx[ba] = s >= 0 ? s - start : 0;
  const int lab = s >= 0 ? w.glab[s] : L.nc;
  labels[ba] = lab;
  const double4 g = s >= 0 ? w.gbox[s] : (cnt > 0 ? w.gbox[start] : make_double4(0.0, 0.0, 0.0, 0.0));
  reinterpret_cast<double4*>(tbox)[ba] = g;
  if (L.mode == CVB_YOLOV6_TAL) {
    double al = 0.0, io = 0.0;
    if (s >= 0) {
      io = iou_calc(g, pd);
      al = tal_metric(class_score(L, scores, ba, lab), io);
      atomicMax(&w.pos_align[s], dkey(al));
      atomicMax(&w.pos_iou[s], dkey(io));
    }
    w.align[ba] = al;
    w.iou[ba] = io;
  }
}

// the soft label (= target_scores.sum(-1)) and the (1 - IoU) term of every anchor; per-CTA fp64 partials of
// (sum w (1 - IoU), sum w, positives, sum pred_distri)
__global__ void __launch_bounds__(kV6Threads) v6_loss_kernel(V6Levels L, const float* __restrict__ distri, V6Ws w, const uint8_t* __restrict__ fg,
                                                             const int32_t* __restrict__ gt_idx, const int32_t* __restrict__ labels,
                                                             const double* __restrict__ tbox, double* __restrict__ score) {
  __shared__ double red[kV6Threads / 32][4];
  const int b = blockIdx.y, a = blockIdx.x * blockDim.x + threadIdx.x;
  double v[4] = {0.0, 0.0, 0.0, 0.0};
  if (a < L.A) {
    const size_t ba = (size_t)b * L.A + a;
    const float4 d = reinterpret_cast<const float4*>(distri)[ba];
    v[3] = (((double)d.x + (double)d.y) + (double)d.z) + (double)d.w;
    double sc = 0.0;
    if (fg[ba]) {
      const Anchor an = anchor_at(L, a);
      const int lab = labels[ba];
      const bool valid = lab >= 0 && lab < L.nc;
      if (L.mode == CVB_YOLOV6_ATSS) {
        // target_scores (fp32) = one_hot * IoU(GT, pred box in pixels), rounded to fp32
        sc = valid ? (double)(float)iou_calc(reinterpret_cast<const double4*>(tbox)[ba], times(pred_box(distri, ba, an), an.s)) : 0.0;
      } else {
        const int s = w.img_start[b] + gt_idx[ba];
        sc = valid ? (w.align[ba] * dkey_value(w.pos_iou[s])) / (dkey_value(w.pos_align[s]) + 1e-9) : 0.0;
      }
      const double4 t = reinterpret_cast<const double4*>(tbox)[ba];
      const double st = (double)an.s;
      const double4 ts = make_double4(t.x / st, t.y / st, t.z / st, t.w / st);
      const D l = box_loss(d, __fdiv_rn(an.sx, an.s), __fdiv_rn(an.sy, an.s), ts, L.siou);
      v[0] = l.v * sc;
      v[1] = sc;
      v[2] = 1.0;
    }
    score[ba] = sc;
  }
  block_sum<kV6Threads>(v, red);
  if (threadIdx.x == 0) {
    double* p = w.partial + ((size_t)b * L.nblk + blockIdx.x) * 4;
#pragma unroll
    for (int k = 0; k < 4; ++k) p[k] = v[k];
  }
}

// stats = (sum w (1 - IoU), target_scores_sum, num_pos, sum pred_distri); L = loss_sum / target_scores_sum (not divided when the sum is
// 0), 0 * sum pred_distri without positives; out = (w_iou L, w_dfl L, w_class L)
__global__ void __launch_bounds__(kV6FinalThreads) v6_final_kernel(V6Levels L, V6Ws w, double* __restrict__ stats, double* __restrict__ out) {
  __shared__ double red[kV6FinalThreads / 32][4];
  double v[4] = {0.0, 0.0, 0.0, 0.0};
  const int n = L.B * L.nblk;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
#pragma unroll
    for (int k = 0; k < 4; ++k) v[k] += w.partial[(size_t)i * 4 + k];
  }
  block_sum<kV6FinalThreads>(v, red);
  if (threadIdx.x != 0) return;
  // ATSS target_scores are fp32, TAL's fp64
  const double S = L.mode == CVB_YOLOV6_ATSS ? (double)(float)v[1] : v[1];
  double loss;
  if (v[2] > 0.0) loss = S == 0.0 ? v[0] : v[0] / S;
  else loss = (double)((float)v[3] * 0.0f);
  stats[0] = v[0];
  stats[1] = S;
  stats[2] = v[2];
  stats[3] = v[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) out[k] = L.wt[k] * loss;
}

// ------------------------------------------------------------------------------------------------------------------ backward
__global__ void __launch_bounds__(kV6Threads) v6_bwd_kernel(V6Levels L, const float* __restrict__ distri, const uint8_t* __restrict__ fg,
                                                            const double* __restrict__ tbox, const double* __restrict__ score,
                                                            const double* __restrict__ stats, const double* __restrict__ gout,
                                                            float* __restrict__ gdistri) {
  const int b = blockIdx.y, a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= L.A) return;
  const size_t ba = (size_t)b * L.A + a;
  float4 r = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
  if (stats[2] > 0.0 && fg[ba]) {
    const double S = stats[1];
    const double g = ((L.wt[0] * gout[0] + L.wt[1] * gout[1]) + L.wt[2] * gout[2]) * score[ba] / (S == 0.0 ? 1.0 : S);
    const Anchor an = anchor_at(L, a);
    const double4 t = reinterpret_cast<const double4*>(tbox)[ba];
    const double st = (double)an.s;
    const double4 ts = make_double4(t.x / st, t.y / st, t.z / st, t.w / st);
    const D l = box_loss(reinterpret_cast<const float4*>(distri)[ba], __fdiv_rn(an.sx, an.s), __fdiv_rn(an.sy, an.s), ts, L.siou);
    r = make_float4((float)(g * l.d[0]), (float)(g * l.d[1]), (float)(g * l.d[2]), (float)(g * l.d[3]));
  }
  reinterpret_cast<float4*>(gdistri)[ba] = r;
}

// ------------------------------------------------------------------------------------------------------------------ host
int make_levels(const char* what, const CvbYolov6LossParams* p, int32_t nt, V6Levels* L) {
  CVB_REQUIRE(p, "%s: params required", what);
  CVB_REQUIRE(p->nlev >= 1 && p->nlev <= CVB_YOLOV6_MAX_LEVELS, "%s: 1 to %d levels supported (got %d)", what, CVB_YOLOV6_MAX_LEVELS, p->nlev);
  CVB_REQUIRE(p->B >= 1 && p->B <= 65535, "%s: batch must be in [1, 65535] (got %d)", what, p->B);
  CVB_REQUIRE(p->nc >= 1 && p->nc <= 65536, "%s: num_classes must be in [1, 65536] (got %d)", what, p->nc);
  CVB_REQUIRE(nt >= 0 && nt <= (1 << 24), "%s: nt must be in [0, 2^24] target rows (got %d)", what, nt);
  CVB_REQUIRE(p->assigner == CVB_YOLOV6_ATSS || p->assigner == CVB_YOLOV6_TAL, "%s: assigner must be CVB_YOLOV6_ATSS or CVB_YOLOV6_TAL (got %d)",
              what, p->assigner);
  CVB_REQUIRE(p->iou_type == CVB_YOLOV6_GIOU || p->iou_type == CVB_YOLOV6_SIOU, "%s: iou_type must be CVB_YOLOV6_GIOU or CVB_YOLOV6_SIOU (got %d)",
              what, p->iou_type);
  CVB_REQUIRE(p->grid_cell_size > 0.0f && p->grid_cell_offset >= 0.0f && p->ori_img_size > 0.0f,
              "%s: grid_cell_size and ori_img_size must be > 0 and grid_cell_offset >= 0", what);
  *L = V6Levels{};
  long long A = 0;
  for (int l = 0; l < p->nlev; ++l) {
    const int h = p->h[l], wd = p->w[l];
    const float s = p->strides[l];
    CVB_REQUIRE(h > 0 && wd > 0 && h <= 65536 && wd <= 65536, "%s: level %d map must be h, w in [1, 65536] (got %d x %d)", what, l, h, wd);
    CVB_REQUIRE(s >= 1.0f && s <= 4096.0f && s == floorf(s), "%s: level %d stride must be a positive integer <= 4096 (got %g)", what, l, (double)s);
    CVB_REQUIRE((double)(h + 1) * s < (double)(1 << 24) && (double)(wd + 1) * s < (double)(1 << 24),
                "%s: level %d map too large for exact fp32 anchor coordinates", what, l);
    L->off[l] = (int)A;
    L->w[l] = wd;
    L->stride[l] = s;
    L->half[l] = (float)((double)p->grid_cell_size * (double)s * 0.5);
    A += (long long)h * wd;
  }
  CVB_REQUIRE((long long)p->B * A < (1LL << 31) / 4, "%s: B x anchors too large (%lld)", what, (long long)p->B * A);
  CVB_REQUIRE(p->assigner != CVB_YOLOV6_TAL || A >= kV6TalK, "%s: the task-aligned assigner needs at least %d anchors (got %lld)", what, kV6TalK, A);
  L->off[p->nlev] = (int)A;
  L->nlev = p->nlev;
  L->A = (int)A;
  L->B = p->B;
  L->nc = p->nc;
  L->nt = nt;
  L->mode = p->assigner;
  L->siou = p->iou_type == CVB_YOLOV6_SIOU;
  L->offset = p->grid_cell_offset;
  L->scale = p->ori_img_size;
  for (int k = 0; k < 3; ++k) L->wt[k] = p->loss_weight[k];
  L->nblk = ceil_div((int)A, kV6Threads);
  return CVB_OK;
}

}  // namespace
}  // namespace cvb

using namespace cvb;

extern "C" size_t cvb_train_yolov6_loss_workspace_bytes(const CvbYolov6LossParams* p, int32_t nt) {
  V6Levels L;
  if (make_levels("train_yolov6_loss_workspace_bytes", p, nt, &L) != CVB_OK) return 0;
  return v6_ws(nullptr, L.B, L.A, nt, L.nblk).bytes;
}

extern "C" int cvb_train_yolov6_loss_fwd(const CvbYolov6LossParams* p, const float* pred_scores, const float* pred_distri, const double* gt, int32_t nt,
                                         uint8_t* fg_mask, int32_t* gt_idx, int32_t* labels, double* target_boxes, double* target_scores,
                                         double* stats, double* out, void* workspace, size_t ws_bytes, void* stream) {
  const char* what = "train_yolov6_loss_fwd";
  V6Levels L;
  const int rc = make_levels(what, p, nt, &L);
  if (rc != CVB_OK) return rc;
  CVB_REQUIRE(pred_scores && pred_distri && is_aligned(pred_scores, 4) && is_aligned(pred_distri, 16),
              "%s: pred_scores (4-byte aligned) and pred_distri (16-byte aligned) are required", what);
  CVB_REQUIRE(nt == 0 || (gt && is_aligned(gt, 8)), "%s: gt (8-byte aligned) is required when nt > 0", what);
  CVB_REQUIRE(fg_mask && gt_idx && labels && target_boxes && target_scores && stats && out,
              "%s: fg_mask, gt_idx, labels, target_boxes, target_scores, stats and out are required", what);
  CVB_REQUIRE(is_aligned(gt_idx, 4) && is_aligned(labels, 4) && is_aligned(target_boxes, 32) && is_aligned(target_scores, 8) && is_aligned(stats, 8) &&
                  is_aligned(out, 8),
              "%s: gt_idx / labels 4-byte, target_boxes 32-byte, target_scores / stats / out 8-byte aligned", what);
  CVB_REQUIRE(workspace && is_aligned(workspace, 256), "%s: workspace required, 256-byte aligned", what);
  const V6Ws w = v6_ws(workspace, L.B, L.A, nt, L.nblk);
  CVB_REQUIRE(ws_bytes >= w.bytes, "%s: workspace of %zu bytes too small (%zu needed)", what, ws_bytes, w.bytes);
  cudaStream_t st = as_stream(stream);
  const dim3 grid(L.nblk, L.B);
  v6_pack_kernel<<<L.B, kV6Threads, 0, st>>>(L, gt, w);
  int n = 1;
  if (nt > 0) {
    const int sel = ceil_div(nt, kV6SelWarps);
    if (L.mode == CVB_YOLOV6_ATSS) v6_atss_select_kernel<<<sel, kV6SelWarps * 32, 0, st>>>(L, w);
    else v6_tal_select_kernel<<<sel, kV6SelWarps * 32, 0, st>>>(L, pred_scores, pred_distri, w);
    ++n;
  }
  v6_resolve_kernel<<<grid, kV6Threads, 0, st>>>(L, pred_scores, pred_distri, w, fg_mask, gt_idx, labels, target_boxes);
  v6_loss_kernel<<<grid, kV6Threads, 0, st>>>(L, pred_distri, w, fg_mask, gt_idx, labels, target_boxes, target_scores);
  v6_final_kernel<<<1, kV6FinalThreads, 0, st>>>(L, w, stats, out);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch(n + 3);
  return CVB_OK;
}

extern "C" int cvb_train_yolov6_loss_bwd(const CvbYolov6LossParams* p, const float* pred_distri, const uint8_t* fg_mask, const double* target_boxes,
                                         const double* target_scores, const double* stats, const double* grad_out, float* grad_distri, void* stream) {
  const char* what = "train_yolov6_loss_bwd";
  V6Levels L;
  const int rc = make_levels(what, p, 0, &L);
  if (rc != CVB_OK) return rc;
  CVB_REQUIRE(pred_distri && grad_distri && is_aligned(pred_distri, 16) && is_aligned(grad_distri, 16),
              "%s: pred_distri and grad_distri are required, 16-byte aligned", what);
  CVB_REQUIRE(fg_mask && target_boxes && target_scores && stats && grad_out && is_aligned(target_boxes, 32) && is_aligned(target_scores, 8) &&
                  is_aligned(stats, 8) && is_aligned(grad_out, 8),
              "%s: fg_mask, target_boxes (32-byte aligned), target_scores, stats and grad_out (8-byte aligned) are required", what);
  v6_bwd_kernel<<<dim3(L.nblk, L.B), kV6Threads, 0, as_stream(stream)>>>(L, pred_distri, fg_mask, target_boxes, target_scores, stats, grad_out,
                                                                          grad_distri);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}
