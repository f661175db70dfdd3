// The FCOS training loss on the device: point assignment (GenTargets), the focal / centerness / GIoU losses and their gradient with
// respect to the head's fp32 NCHW outputs (src/losses/fcos_loss.py; the algorithm is restated in oracle/fcos_loss_oracle.py).
//
// Forward (cvb_train_fcos_loss_fwd), all stream-ordered, no host sync, CUDA-graph capturable:
//   1. fcos_assign_kernel  one thread per (image, point), the image's GT boxes staged in shared memory: the first area minimum over the
//                          positive (point, GT) pairs -> matched_gt, and the point's centerness BCE and 1 - GIoU, summed per CTA in fp64.
//   2. fcos_focal_kernel   one thread per (image, point, chunk of 16 classes): the sigmoid focal loss of every logit, read coalesced along
//                          h w; the target class comes from matched_gt.  fp64 per-CTA partials.
//   3. fcos_final_kernel   one CTA, one warp per image: each image's partials in a fixed order, num_pos, and the four outputs.
// Backward (cvb_train_fcos_loss_bwd): fcos_bwd_kernel, with the focal kernel's grid, writes every element of the class-logit gradients; its
// first class chunk also writes the centerness and regression gradients of its points.  No float atomics: results are bitwise reproducible.
//
// Precision: every assignment quantity is one correctly rounded fp32 operation in the reference's order (this file is compiled with
// --fmad=false), so the targets are bitwise the reference's.  The focal and GIoU gradients follow torch.autograd's chain in fp32, with its
// rules at the kinks: torch.min / torch.max split the gradient evenly on a tie, clamp(min) passes it at the bound, and a pt of 0 gives an
// inf loss and a NaN gradient.  The loss sums are accumulated in fp64.
#include <limits.h>

#include "internal.h"

namespace cvb {
namespace {

constexpr int kFcosMaxLevels = 8;
constexpr int kFcosMaxGt = 1024;      // GT rows per image (boxes [B, m, 4])
constexpr int kFcosThreads = 256;
constexpr int kFcosClsChunk = 16;     // classes per thread in the focal passes
constexpr int kFcosFinalThreads = 1024;  // one warp per image
constexpr float kFcosNotPos = 99999999.0f;  // the area given to a (point, GT) pair that is not positive

struct FcosLevels {
  const float* cls[kFcosMaxLevels];  // [B, nc, h, w]
  const float* cnt[kFcosMaxLevels];  // [B, 1, h, w]
  const float* reg[kFcosMaxLevels];  // [B, 4, h, w]
  float* gcls[kFcosMaxLevels];       // gradients, same shapes (backward only)
  float* gcnt[kFcosMaxLevels];
  float* greg[kFcosMaxLevels];
  int w[kFcosMaxLevels], hw[kFcosMaxLevels];
  int off[kFcosMaxLevels + 1];       // first point of each level; off[nlev] = A
  int stride[kFcosMaxLevels];
  float lo[kFcosMaxLevels], hi[kFcosMaxLevels], radius[kFcosMaxLevels];
  int nlev, A, nc, B, m, nblk, nchunk;
};

struct Point {
  int l, i, hw;  // level, index within the level's h w, h w
  float x, y;    // image coordinates: column * stride + stride / 2
};

__device__ __forceinline__ Point point_at(const FcosLevels& L, int a) {
  Point r{0, 0, 1, 0.0f, 0.0f};
#pragma unroll
  for (int l = 0; l < kFcosMaxLevels; ++l) {
    if (l < L.nlev && a >= L.off[l] && a < L.off[l + 1]) {
      const int i = a - L.off[l], s = L.stride[l];
      r.l = l;
      r.i = i;
      r.hw = L.hw[l];
      r.x = (float)((i % L.w[l]) * s) + (float)(s / 2);
      r.y = (float)((i / L.w[l]) * s) + (float)(s / 2);
    }
  }
  return r;
}

// (l, t, r, b) offsets of the point from a GT box (x1, y1, x2, y2)
__device__ __forceinline__ float4 ltrb(float4 g, float x, float y) { return make_float4(x - g.x, y - g.y, g.z - x, g.w - y); }

// The matched GT row of a point (-1 = background): the first minimum over the m rows of the area, with kFcosNotPos for a pair that is not
// positive (inside the box, max offset in the level's range, centre offset below the radius).  Every test is the reference's fp32 compare.
__device__ __forceinline__ int match_point(const float4* gts, int m, float x, float y, float lo, float hi, float radius) {
  float best = 0.0f;
  int arg = 0;
  bool any = false;
  for (int g = 0; g < m; ++g) {
    const float4 b = gts[g];
    const float4 o = ltrb(b, x, y);
    const bool inside = o.x > 0.0f && o.y > 0.0f && o.z > 0.0f && o.w > 0.0f;  // min(l, t, r, b) > 0 (NaN: false)
    const float omax = fmaxf(fmaxf(o.x, o.y), fmaxf(o.z, o.w));               // (no NaN once inside)
    const float cx = (b.x + b.z) / 2.0f, cy = (b.y + b.w) / 2.0f;
    const float cmax = fmaxf(fmaxf(x - cx, y - cy), fmaxf(cx - x, cy - y));
    const bool pos = inside && omax > lo && omax <= hi && cmax < radius;
    const float area = pos ? (o.x + o.z) * (o.y + o.w) : kFcosNotPos;
    if (g == 0 || area < best) { best = area; arg = g; }
    any = any || pos;
  }
  return any ? arg : -1;
}

// sqrt((min(l, r) min(t, b)) / (max(l, r) max(t, b) + 1e-10))
__device__ __forceinline__ float centerness(float4 o) {
  return sqrtf((fminf(o.x, o.z) * fminf(o.y, o.w)) / (fmaxf(o.x, o.z) * fmaxf(o.y, o.w) + 1e-10f));
}

// torch.min / torch.max / clamp(min) of fp32 values, NaN-propagating as torch is
__device__ __forceinline__ float tmin(float a, float b) { return (a != a || b != b) ? a + b : fminf(a, b); }
__device__ __forceinline__ float tmax(float a, float b) { return (a != a || b != b) ? a + b : fmaxf(a, b); }
__device__ __forceinline__ float clamp_lo(float v, float lo) { return v < lo ? lo : v; }

// 1 - GIoU of an ltrb prediction against its ltrb target (giou_loss, G_area.clamp(1e-10))
__device__ __forceinline__ float giou_loss(float4 p, float4 t) {
  const float w = clamp_lo(tmin(p.z, t.z) + tmin(p.x, t.x), 0.0f), h = clamp_lo(tmin(p.w, t.w) + tmin(p.y, t.y), 0.0f);
  const float ov = w * h;
  const float a1 = (p.z + p.x) * (p.w + p.y), a2 = (t.z + t.x) * (t.w + t.y);
  const float u = (a1 + a2) - ov;
  const float iou = ov / u;
  const float W = clamp_lo(tmax(p.z, t.z) + tmax(p.x, t.x), 0.0f), H = clamp_lo(tmax(p.w, t.w) + tmax(p.y, t.y), 0.0f);
  const float G = W * H;
  return 1.0f - (iou - (G - u) / clamp_lo(G, 1e-10f));
}

// share of a torch.min(a, b) / torch.max(a, b) gradient that goes to a: all, half on a tie, none
__device__ __forceinline__ float min_share(float a, float b) { return a < b ? 1.0f : (a == b ? 0.5f : 0.0f); }
__device__ __forceinline__ float max_share(float a, float b) { return a > b ? 1.0f : (a == b ? 0.5f : 0.0f); }

// d(gl (1 - GIoU)) / d(p), along autograd's chain through giou_loss
__device__ __forceinline__ float4 giou_grad(float4 p, float4 t, float gl) {
  const float wr = tmin(p.z, t.z) + tmin(p.x, t.x), hr = tmin(p.w, t.w) + tmin(p.y, t.y);
  const float w = clamp_lo(wr, 0.0f), h = clamp_lo(hr, 0.0f);
  const float ov = w * h;
  const float sw = p.z + p.x, sh = p.w + p.y;
  const float a1 = sw * sh, a2 = (t.z + t.x) * (t.w + t.y);
  const float u = (a1 + a2) - ov;
  const float Wr = tmax(p.z, t.z) + tmax(p.x, t.x), Hr = tmax(p.w, t.w) + tmax(p.y, t.y);
  const float W = clamp_lo(Wr, 0.0f), H = clamp_lo(Hr, 0.0f);
  const float G = W * H, Gc = clamp_lo(G, 1e-10f), N = G - u;
  // loss = 1 - iou + N / Gc, iou = ov / u, N = G - u, u = a1 + a2 - ov
  const float g_iou = -gl;
  const float gN = gl / Gc;
  const float gG = gN + (G >= 1e-10f ? -gl * ((N / Gc) / Gc) : 0.0f);
  const float gu = -gN + -g_iou * ((ov / u) / u);
  const float g_ov = g_iou / u - gu;
  const float gw = wr >= 0.0f ? g_ov * h : 0.0f, gh = hr >= 0.0f ? g_ov * w : 0.0f;
  const float gW = Wr >= 0.0f ? gG * H : 0.0f, gH = Hr >= 0.0f ? gG * W : 0.0f;
  return make_float4(gw * min_share(p.x, t.x) + gW * max_share(p.x, t.x) + gu * sh, gh * min_share(p.y, t.y) + gH * max_share(p.y, t.y) + gu * sw,
                     gw * min_share(p.z, t.z) + gW * max_share(p.z, t.z) + gu * sh, gh * min_share(p.w, t.w) + gH * max_share(p.w, t.w) + gu * sw);
}

// Sigmoid focal loss (alpha 0.25, gamma 2) of one logit against a 0 / 1 target: p = sigmoid(x), pt = p t + (1 - p)(1 - t),
// w = 0.25 t + 0.75 (1 - t), -w (1 - pt)^2 log(pt).  With t in {0, 1} pt is p or 1 - p and w is 0.25 or 0.75 exactly.
__device__ __forceinline__ float focal(float x, bool pos) {
  const float p = sigmoidf(x);
  const float pt = pos ? p : 1.0f - p;
  const float q = 1.0f - pt;
  return (-(pos ? 0.25f : 0.75f) * (q * q)) * logf(pt);
}

// g d(focal)/dx along autograd's chain: the log's 1 / pt, the square's 2 (1 - pt), the unused branch of pt multiplied by 0, and the sigmoid's
// p (1 - p).  A pt of 0 (or a 1 / pt that overflows) therefore gives NaN, as in the reference.
__device__ __forceinline__ float focal_grad(float x, bool pos, float g) {
  const float p = sigmoidf(x);
  const float pt = pos ? p : 1.0f - p;
  const float q = 1.0f - pt;
  const float nw = -(pos ? 0.25f : 0.75f);
  const float g_pt = (g * (nw * (q * q))) / pt - ((g * logf(pt)) * nw) * (2.0f * q);
  const float g_p = pos ? g_pt * 1.0f - g_pt * 0.0f : g_pt * 0.0f - g_pt * 1.0f;
  return (g_p * (1.0f - p)) * p;
}

// class index of a point's one-hot row (-1: none): the matched GT's label - 1 when the label is in 1..nc
__device__ __forceinline__ int target_class(const FcosLevels& L, const int32_t* labels, int b, int mg) {
  if (mg < 0) return -1;
  const int lab = labels[(size_t)b * L.m + mg];
  return (lab >= 1 && lab <= L.nc) ? lab - 1 : -1;
}

// --------------------------------------------------------------------------------------------------------------------------- forward
__global__ void __launch_bounds__(kFcosThreads) fcos_assign_kernel(FcosLevels L, const float* __restrict__ boxes, int32_t* __restrict__ matched_gt,
                                                                   float* __restrict__ tgt, double* __restrict__ partial) {
  extern __shared__ float4 gts[];
  __shared__ double red[kFcosThreads / 32][3];
  const int b = blockIdx.y;
  for (int g = threadIdx.x; g < L.m; g += blockDim.x) gts[g] = reinterpret_cast<const float4*>(boxes)[(size_t)b * L.m + g];
  __syncthreads();
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  double v[3] = {0.0, 0.0, 0.0};  // centerness BCE, 1 - GIoU, positives
  if (a < L.A) {
    const Point pt = point_at(L, a);
    const int mg = match_point(gts, L.m, pt.x, pt.y, L.lo[pt.l], L.hi[pt.l], L.radius[pt.l]);
    matched_gt[(size_t)b * L.A + a] = mg;
    float t[5] = {-1.0f, -1.0f, -1.0f, -1.0f, -1.0f};  // centerness, l, t, r, b targets (-1: background)
    if (mg >= 0) {
      const float4 o = ltrb(gts[mg], pt.x, pt.y);
      const size_t base = (size_t)b * pt.hw + pt.i;
      t[0] = centerness(o);
      t[1] = o.x;
      t[2] = o.y;
      t[3] = o.z;
      t[4] = o.w;
      v[0] = bce_logits(L.cnt[pt.l][base], t[0]);
      const float* r = L.reg[pt.l] + (size_t)b * 4 * pt.hw + pt.i;
      v[1] = giou_loss(make_float4(r[0], r[pt.hw], r[2 * pt.hw], r[3 * pt.hw]), o);
      v[2] = 1.0;
    }
    if (tgt) {
#pragma unroll
      for (int k = 0; k < 5; ++k) tgt[((size_t)b * L.A + a) * 5 + k] = t[k];
    }
  }
  block_sum<kFcosThreads>(v, red);
  if (threadIdx.x == 0) {
    double* d = partial + ((size_t)b * L.nblk + blockIdx.x) * 3;
    d[0] = v[0];
    d[1] = v[1];
    d[2] = v[2];
  }
}

__global__ void __launch_bounds__(kFcosThreads) fcos_focal_kernel(FcosLevels L, const int32_t* __restrict__ labels, const int32_t* __restrict__ matched_gt,
                                                                  double* __restrict__ partial) {
  __shared__ double red[kFcosThreads / 32][1];
  const int b = blockIdx.z, c0 = blockIdx.y * kFcosClsChunk;
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  double v[1] = {0.0};
  if (a < L.A) {
    const Point pt = point_at(L, a);
    const int k = target_class(L, labels, b, matched_gt[(size_t)b * L.A + a]);
    const float* x = L.cls[pt.l] + (size_t)b * L.nc * pt.hw + pt.i;
    const int c1 = min(c0 + kFcosClsChunk, L.nc);
    float e[kFcosClsChunk];
#pragma unroll
    for (int j = 0; j < kFcosClsChunk; ++j) e[j] = c0 + j < c1 ? x[(size_t)(c0 + j) * pt.hw] : 0.0f;
#pragma unroll
    for (int j = 0; j < kFcosClsChunk; ++j)
      if (c0 + j < c1) v[0] += focal(e[j], c0 + j == k);
  }
  block_sum<kFcosThreads>(v, red);
  if (threadIdx.x == 0) partial[((size_t)b * L.nchunk + blockIdx.y) * L.nblk + blockIdx.x] = v[0];
}

// Each image's sums in a fixed order, one warp per image; out = (cls, cnt, reg, total) with every term the batch mean of
// sum_b / max(num_pos_b, 1), the images added in order by thread 0.
__global__ void __launch_bounds__(kFcosFinalThreads) fcos_final_kernel(FcosLevels L, const double* __restrict__ pt_partial,
                                                                       const double* __restrict__ cls_partial, int32_t* __restrict__ num_pos,
                                                                       float* __restrict__ out) {
  __shared__ double img[kFcosFinalThreads / 32][3];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int nf = L.nchunk * L.nblk;
  double acc[3] = {0.0, 0.0, 0.0};
  for (int b0 = 0; b0 < L.B; b0 += kFcosFinalThreads / 32) {
    const int b = b0 + wid;
    if (b < L.B) {
      double v[4] = {0.0, 0.0, 0.0, 0.0};  // focal, centerness, GIoU, positives
      for (int i = lane; i < nf; i += 32) v[0] += cls_partial[(size_t)b * nf + i];
      for (int i = lane; i < L.nblk; i += 32) {
        const double* d = pt_partial + ((size_t)b * L.nblk + i) * 3;
        v[1] += d[0];
        v[2] += d[1];
        v[3] += d[2];
      }
#pragma unroll
      for (int k = 0; k < 4; ++k) v[k] = warp_sum(v[k]);
      if (lane == 0) {
        const double np = fmax(v[3], 1.0);
        img[wid][0] = v[0] / np;
        img[wid][1] = v[1] / np;
        img[wid][2] = v[2] / np;
        num_pos[b] = (int32_t)v[3];
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 0; w < kFcosFinalThreads / 32 && b0 + w < L.B; ++w) {
        acc[0] += img[w][0];
        acc[1] += img[w][1];
        acc[2] += img[w][2];
      }
    }
    __syncthreads();  // (img is reused by the next images)
  }
  if (threadIdx.x == 0) {
    const float c = (float)(acc[0] / L.B), n = (float)(acc[1] / L.B), r = (float)(acc[2] / L.B);
    out[0] = c;
    out[1] = n;
    out[2] = r;
    out[3] = (c + n) + r;
  }
}

// --------------------------------------------------------------------------------------------------------------------------- backward
__global__ void __launch_bounds__(kFcosThreads) fcos_bwd_kernel(FcosLevels L, const float* __restrict__ boxes, const int32_t* __restrict__ labels,
                                                                const int32_t* __restrict__ matched_gt, const int32_t* __restrict__ num_pos,
                                                                const float* __restrict__ gout) {
  const int b = blockIdx.z, c0 = blockIdx.y * kFcosClsChunk;
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= L.A) return;
  const Point pt = point_at(L, a);
  const int mg = matched_gt[(size_t)b * L.A + a];
  // total = cls + cnt + reg, each also an output of its own: d/d(term) = g_term + g_total; then the mean over B and the division by num_pos
  const float np = (float)max(num_pos[b], 1), fB = (float)L.B;
  const float s_cls = ((gout[0] + gout[3]) / fB) / np;
  const int k = target_class(L, labels, b, mg);
  const size_t cbase = (size_t)b * L.nc * pt.hw + pt.i;
  const float* x = L.cls[pt.l] + cbase;
  float* gx = L.gcls[pt.l] + cbase;
  const int c1 = min(c0 + kFcosClsChunk, L.nc);
  float e[kFcosClsChunk];
#pragma unroll
  for (int j = 0; j < kFcosClsChunk; ++j) e[j] = c0 + j < c1 ? x[(size_t)(c0 + j) * pt.hw] : 0.0f;
#pragma unroll
  for (int j = 0; j < kFcosClsChunk; ++j)
    if (c0 + j < c1) gx[(size_t)(c0 + j) * pt.hw] = focal_grad(e[j], c0 + j == k, s_cls);
  if (blockIdx.y != 0) return;
  const size_t base = (size_t)b * pt.hw + pt.i, rbase = (size_t)b * 4 * pt.hw + pt.i;
  float* gc = L.gcnt[pt.l] + base;
  float* gr = L.greg[pt.l] + rbase;
  if (mg < 0) {
    *gc = 0.0f;
#pragma unroll
    for (int j = 0; j < 4; ++j) gr[(size_t)j * pt.hw] = 0.0f;
    return;
  }
  const float4 o = ltrb(reinterpret_cast<const float4*>(boxes)[(size_t)b * L.m + mg], pt.x, pt.y);
  const float s_cnt = ((gout[1] + gout[3]) / fB) / np, s_reg = ((gout[2] + gout[3]) / fB) / np;
  *gc = (sigmoidf(L.cnt[pt.l][base]) - centerness(o)) * s_cnt;
  const float* r = L.reg[pt.l] + rbase;
  const float4 d = giou_grad(make_float4(r[0], r[pt.hw], r[2 * pt.hw], r[3 * pt.hw]), o, s_reg);
  gr[0] = d.x;
  gr[pt.hw] = d.y;
  gr[2 * (size_t)pt.hw] = d.z;
  gr[3 * (size_t)pt.hw] = d.w;
}

// --------------------------------------------------------------------------------------------------------------------------- host
struct FcosWs {
  double *pt_partial, *cls_partial;
  size_t bytes;
};

inline int point_blocks(int A) { return ceil_div(A, kFcosThreads); }
inline int class_chunks(int nc) { return ceil_div(nc, kFcosClsChunk); }

FcosWs fcos_ws(void* base, int B, int A, int nc) {
  WsCarver c(base);
  FcosWs w{};
  const size_t nb = (size_t)B * point_blocks(A);
  w.pt_partial = static_cast<double*>(c.take(nb * 3 * sizeof(double)));
  w.cls_partial = static_cast<double*>(c.take(nb * class_chunks(nc) * sizeof(double)));
  w.bytes = c.bytes();
  return w;
}

// Validates the description shared by the forward and the backward and fills L (gradients: may be NULL in the forward).
int make_levels(const char* what, const float* const* cls, const float* const* cnt, const float* const* reg, const int32_t* shapes, const float* strides,
                const float* limit_range, int32_t nlev, const float* boxes, const int32_t* labels, int32_t B, int32_t m, float* const* gcls,
                float* const* gcnt, float* const* greg, FcosLevels* L) {
  CVB_REQUIRE(cls && cnt && reg && shapes && strides && limit_range, "%s: cls, cnt, reg, shapes, strides and limit_range are required", what);
  CVB_REQUIRE(nlev >= 1 && nlev <= kFcosMaxLevels, "%s: 1 to %d levels supported (got %d)", what, kFcosMaxLevels, nlev);
  CVB_REQUIRE(B >= 1, "%s: batch must be >= 1 (got %d)", what, B);
  CVB_REQUIRE(m >= 0 && m <= kFcosMaxGt, "%s: m must be in [0, %d] GT rows per image (got %d)", what, kFcosMaxGt, m);
  if (m > 0)
    CVB_REQUIRE(boxes && labels && is_aligned(boxes, 16) && is_aligned(labels, 4), "%s: boxes (16-byte aligned) and labels (4-byte aligned) are required", what);
  const int nc = shapes[1];
  CVB_REQUIRE(nc >= 1 && nc <= 65536, "%s: num_classes must be in [1, 65536] (got %d)", what, nc);
  *L = FcosLevels{};
  long long A = 0;
  for (int l = 0; l < nlev; ++l) {
    const int32_t* c = shapes + 12 * l;
    const int32_t *n = c + 4, *r = c + 8;
    CVB_REQUIRE(c[0] == B && c[1] == nc && c[2] > 0 && c[3] > 0, "%s: level %d cls_logits must be [B=%d, num_classes=%d, h > 0, w > 0] (got [%d, %d, %d, %d])",
                what, l, B, nc, c[0], c[1], c[2], c[3]);
    CVB_REQUIRE(n[0] == B && n[1] == 1 && n[2] == c[2] && n[3] == c[3], "%s: level %d cnt_logits must be [B=%d, 1, %d, %d] (got [%d, %d, %d, %d])", what, l,
                B, c[2], c[3], n[0], n[1], n[2], n[3]);
    CVB_REQUIRE(r[0] == B && r[1] == 4 && r[2] == c[2] && r[3] == c[3], "%s: level %d reg_preds must be [B=%d, 4, %d, %d] (got [%d, %d, %d, %d])", what, l,
                B, c[2], c[3], r[0], r[1], r[2], r[3]);
    const float s = strides[l];
    CVB_REQUIRE(s >= 1.0f && s <= 65536.0f && s == floorf(s), "%s: level %d stride must be a positive integer (got %g)", what, l, (double)s);
    const float lo = limit_range[2 * l], hi = limit_range[2 * l + 1];
    CVB_REQUIRE(lo < hi, "%s: level %d limit range must have lo < hi (got [%g, %g])", what, l, (double)lo, (double)hi);
    CVB_REQUIRE(cls[l] && cnt[l] && reg[l] && is_aligned(cls[l], 4) && is_aligned(cnt[l], 4) && is_aligned(reg[l], 4),
                "%s: level %d output missing or not 4-byte aligned", what, l);
    if (gcls)
      CVB_REQUIRE(gcls[l] && gcnt[l] && greg[l] && is_aligned(gcls[l], 4) && is_aligned(gcnt[l], 4) && is_aligned(greg[l], 4),
                  "%s: level %d gradient missing or not 4-byte aligned", what, l);
    CVB_REQUIRE((long long)c[2] * c[3] * s < (1LL << 24) && (long long)c[2] * s < (1LL << 24) && (long long)c[3] * s < (1LL << 24),
                "%s: level %d map too large for exact fp32 point coordinates", what, l);
    CVB_REQUIRE((long long)B * nc * c[2] * c[3] < (1LL << 40), "%s: level %d too large", what, l);
    L->cls[l] = cls[l];
    L->cnt[l] = cnt[l];
    L->reg[l] = reg[l];
    if (gcls) {
      L->gcls[l] = gcls[l];
      L->gcnt[l] = gcnt[l];
      L->greg[l] = greg[l];
    }
    L->w[l] = c[3];
    L->hw[l] = c[2] * c[3];
    L->off[l] = (int)A;
    L->stride[l] = (int)s;
    L->lo[l] = lo;
    L->hi[l] = hi;
    L->radius[l] = (float)((double)s * 1.5);
    A += (long long)c[2] * c[3];
    CVB_REQUIRE(A < INT_MAX, "%s: too many points (%lld)", what, A);
  }
  CVB_REQUIRE((long long)B * A < INT_MAX, "%s: B x points too large (%lld)", what, (long long)B * A);
  CVB_REQUIRE(B <= 65535, "%s: batch must be <= 65535 (got %d)", what, B);
  L->off[nlev] = (int)A;
  L->nlev = nlev;
  L->A = (int)A;
  L->nc = nc;
  L->B = B;
  L->m = m;
  L->nblk = point_blocks((int)A);
  L->nchunk = class_chunks(nc);
  return CVB_OK;
}

}  // namespace
}  // namespace cvb

using namespace cvb;

extern "C" size_t cvb_train_fcos_loss_workspace_bytes(int32_t B, int32_t A, int32_t nc) {
  if (B <= 0 || A <= 0 || nc <= 0) return 0;
  return fcos_ws(nullptr, B, A, nc).bytes;
}

extern "C" int cvb_train_fcos_loss_fwd(const float* const* cls, const float* const* cnt, const float* const* reg, const int32_t* shapes, const float* strides,
                                       const float* limit_range, int32_t nlev, const float* boxes, const int32_t* labels, int32_t B, int32_t m,
                                       int32_t* matched_gt, int32_t* num_pos, float* targets, float* out, void* workspace, size_t ws_bytes,
                                       void* stream) {
  FcosLevels L;
  const int rc = make_levels("train_fcos_loss_fwd", cls, cnt, reg, shapes, strides, limit_range, nlev, boxes, labels, B, m, nullptr, nullptr, nullptr, &L);
  if (rc != CVB_OK) return rc;
  CVB_REQUIRE(matched_gt && num_pos && out && is_aligned(matched_gt, 4) && is_aligned(num_pos, 4) && is_aligned(out, 4),
              "train_fcos_loss_fwd: matched_gt, num_pos and out are required, 4-byte aligned");
  CVB_REQUIRE(is_aligned(targets, 4), "train_fcos_loss_fwd: targets must be 4-byte aligned");
  const FcosWs w = fcos_ws(workspace, B, L.A, L.nc);
  CVB_REQUIRE(workspace && is_aligned(workspace, 256), "train_fcos_loss_fwd: workspace required, 256-byte aligned");
  CVB_REQUIRE(ws_bytes >= w.bytes, "train_fcos_loss_fwd: workspace of %zu bytes too small (%zu needed)", ws_bytes, w.bytes);
  cudaStream_t st = as_stream(stream);
  fcos_assign_kernel<<<dim3(L.nblk, B), kFcosThreads, (size_t)m * sizeof(float4), st>>>(L, boxes, matched_gt, targets, w.pt_partial);
  fcos_focal_kernel<<<dim3(L.nblk, L.nchunk, B), kFcosThreads, 0, st>>>(L, labels, matched_gt, w.cls_partial);
  fcos_final_kernel<<<1, kFcosFinalThreads, 0, st>>>(L, w.pt_partial, w.cls_partial, num_pos, out);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch(3);
  return CVB_OK;
}

extern "C" int cvb_train_fcos_loss_bwd(const float* const* cls, const float* const* cnt, const float* const* reg, const int32_t* shapes, const float* strides,
                                       const float* limit_range, int32_t nlev, const float* boxes, const int32_t* labels, int32_t B, int32_t m,
                                       const int32_t* matched_gt, const int32_t* num_pos, const float* grad_out, float* const* gcls, float* const* gcnt,
                                       float* const* greg, void* stream) {
  CVB_REQUIRE(gcls && gcnt && greg, "train_fcos_loss_bwd: gcls, gcnt and greg are required");
  FcosLevels L;
  const int rc = make_levels("train_fcos_loss_bwd", cls, cnt, reg, shapes, strides, limit_range, nlev, boxes, labels, B, m, gcls, gcnt, greg, &L);
  if (rc != CVB_OK) return rc;
  CVB_REQUIRE(matched_gt && num_pos && grad_out && is_aligned(matched_gt, 4) && is_aligned(num_pos, 4) && is_aligned(grad_out, 4),
              "train_fcos_loss_bwd: matched_gt, num_pos and grad_out are required, 4-byte aligned");
  fcos_bwd_kernel<<<dim3(L.nblk, L.nchunk, B), kFcosThreads, 0, as_stream(stream)>>>(L, boxes, labels, matched_gt, num_pos, grad_out);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}
