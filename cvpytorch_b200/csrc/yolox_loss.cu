// The YOLOX training loss on the device: SimOTA label assignment, the IoU / objectness / class losses and their gradient with respect to
// the head's three fp32 NCHW outputs (src/losses/det/yolox_loss.py:73-436; the algorithm is restated in oracle/yolox_loss_oracle.py).
//
// Forward (cvb_train_yolox_loss_fwd), all stream-ordered, no host sync, CUDA-graph capturable:
//   1. loss_prep_kernel     one CTA per image: nlabel = number of target rows with a positive sum (the image uses its first nlabel rows).
//   2. loss_anchor_kernel   one thread per anchor: decode, sigmoid(obj), the per-anchor class-cost sum S and the candidate flag (strictly
//                           inside any GT box or any GT centre +- 2.5 stride), against the image's GTs staged in shared memory.
//   3. loss_compact_kernel  one CTA per image: the candidate anchors in anchor order.
//   4. loss_gt_kernel       one CTA per (GT, image): IoU and cost over the image's candidates, the top-10 IoUs (dynamic k) and the k
//                           lowest costs (ties: the lower anchor index), kept per thread in registers and merged across the CTA.
//   5. loss_resolve_kernel  one thread per anchor: an anchor taken by several GTs goes to the argmin of its cost over all GTs (ties: the
//                           lower GT index); the matched GT / IoU and the anchor's three loss terms, summed per CTA (block_sum).
//   6. loss_final_kernel    one CTA: the CTA partials by a halving tree (DESIGN.md 2) -> loss, iou_loss, conf_loss, cls_loss, num_fg ratio, num_fg.
// Backward (cvb_train_yolox_loss_bwd): loss_bwd_kernel, one thread per anchor, writes every channel of the fp32 NCHW gradients from the
// saved assignment, scaled by the incoming gradients of the four loss outputs.  No float atomics anywhere: results are bitwise reproducible.
//
// Precision: fp32 in the reference's operation order (this file is compiled with --fmad=false so that no multiply-add is contracted),
// except the class cost, which is re-associated as S(anchor) + a per-GT correction (see cost()).  The loss sums are accumulated in fp64.
#include <float.h>
#include <limits.h>

#include "internal.h"

namespace cvb {
namespace {

constexpr int kLossMaxGt = 1024;   // GT rows per image (targets [B, max_gt, 5])
constexpr int kLossMaxLevels = 4;
constexpr int kTopK = 10;          // n_candidate_k of the dynamic k, and its upper bound
constexpr int kLossThreads = 256;

struct LossLevels {
  const float* p[kLossMaxLevels];  // [B, 5 + nc, h, w] fp32
  float* g[kLossMaxLevels];        // gradients, same shapes (backward only)
  int h[kLossMaxLevels], w[kLossMaxLevels];
  int off[kLossMaxLevels + 1];     // first anchor of each level; off[nlev] = A
  float s[kLossMaxLevels];
  int nlev, A, nc, G;
};

struct Anchor {
  const float* p;  // channel 0 of this anchor: channel c is p[c * hw]
  float* g;
  int hw;
  float x, y, s;   // grid column / row on the (padded) map, stride
};

__device__ __forceinline__ Anchor anchor_at(const LossLevels& L, int b, int a) {
  Anchor r{};
#pragma unroll
  for (int l = 0; l < kLossMaxLevels; ++l) {
    if (l < L.nlev && a >= L.off[l] && a < L.off[l + 1]) {
      const int i = a - L.off[l], hw = L.h[l] * L.w[l];
      const size_t base = (size_t)b * (5 + L.nc) * hw + i;
      r.p = L.p[l] + base;
      r.g = L.g[l] ? L.g[l] + base : nullptr;
      r.hw = hw;
      r.x = (float)(i % L.w[l]);
      r.y = (float)(i / L.w[l]);
      r.s = L.s[l];
    }
  }
  return r;
}

// F.binary_cross_entropy with target 0 / 1: -max(log1p(-q), -100) / -max(log(q), -100)
__device__ __forceinline__ float bce0(float q) { return -fmaxf(log1pf(-q), -100.0f); }
__device__ __forceinline__ float bce1(float q) { return -fmaxf(logf(q), -100.0f); }

// decoded prediction (yolox_loss.py:150-152): xy = (p + grid) * s, wh = exp(p) * s
__device__ __forceinline__ float4 decode(const Anchor& an) {
  return make_float4((an.p[0] + an.x) * an.s, (an.p[an.hw] + an.y) * an.s, expf(an.p[2 * an.hw]) * an.s, expf(an.p[3 * an.hw]) * an.s);
}

__device__ __forceinline__ float4 load_gt(const float* targets, int b, int g, int G, int* cls) {
  const float* r = targets + ((size_t)b * G + g) * 5;
  *cls = (int)r[0];
  return make_float4(r[1], r[2], r[3], r[4]);
}

// in_box / in_center of one GT (cx, cy, w, h) for the anchor centre (xc, yc) (yolox_loss.py:350-403)
__device__ __forceinline__ bool in_box(float4 gt, float xc, float yc) {
  const float l = gt.x - 0.5f * gt.z, r = gt.x + 0.5f * gt.z, t = gt.y - 0.5f * gt.w, bo = gt.y + 0.5f * gt.w;
  return (xc - l) > 0.0f && (yc - t) > 0.0f && (r - xc) > 0.0f && (bo - yc) > 0.0f;
}
__device__ __forceinline__ bool in_center(float4 gt, float xc, float yc, float s) {
  const float rad = 2.5f * s;
  const float l = gt.x - rad, r = gt.x + rad, t = gt.y - rad, bo = gt.y + rad;
  return (xc - l) > 0.0f && (yc - t) > 0.0f && (r - xc) > 0.0f && (bo - yc) > 0.0f;
}

// bboxes_iou(gt, pred, xyxy=False) (yolox_loss.py:14-31)
__device__ __forceinline__ float pair_iou(float4 a, float4 b) {
  const float tlx = fmaxf(a.x - a.z / 2.0f, b.x - b.z / 2.0f), tly = fmaxf(a.y - a.w / 2.0f, b.y - b.w / 2.0f);
  const float brx = fminf(a.x + a.z / 2.0f, b.x + b.z / 2.0f), bry = fminf(a.y + a.w / 2.0f, b.y + b.w / 2.0f);
  const float area_a = a.z * a.w, area_b = b.z * b.w;
  const float en = (tlx < brx && tly < bry) ? 1.0f : 0.0f;
  const float area_i = (brx - tlx) * (bry - tly) * en;
  return area_i / (area_a + area_b - area_i);
}

struct AnchorCost {
  float4 box;   // decoded prediction
  float S;      // sum over classes of BCE(q_c, 0), q_c = sqrt(sigmoid(cls_c) * sigmoid(obj))
  float so;     // sigmoid(obj)
};

// cost(gt, anchor) = cls_cost + 3 (-log(iou + 1e-8)) + 1e5 (not in_box_and_center) (yolox_loss.py:319-335).  The class cost
// sum_c BCE(q_c, onehot_c) is re-associated as S + (BCE(q_k, 1) - BCE(q_k, 0)) with k the GT class (a class outside [0, nc) has no
// one-hot entry: cost S).  Shared by the GT pass and the conflict pass so that both see the same fp32 bits.
__device__ __forceinline__ float cost(const LossLevels& L, const Anchor& an, const AnchorCost& ac, float4 gt, int cls, float* iou_out) {
  const float iou = pair_iou(gt, ac.box);
  float c = ac.S;
  if (cls >= 0 && cls < L.nc) {
    const float q = sqrtf(sigmoidf(an.p[(5 + cls) * an.hw]) * ac.so);
    c = (c - bce0(q)) + bce1(q);
  }
  const float xc = an.x * an.s + 0.5f * an.s, yc = an.y * an.s + 0.5f * an.s;
  const bool both = in_box(gt, xc, yc) && in_center(gt, xc, yc, an.s);
  *iou_out = iou;
  return c + 3.0f * (-logf(iou + 1e-8f)) + 100000.0f * (both ? 0.0f : 1.0f);
}

__device__ __forceinline__ AnchorCost load_cost(const float4* box, const float2* sc, size_t idx) {
  const float2 v = sc[idx];
  return AnchorCost{box[idx], v.x, v.y};
}

// --------------------------------------------------------------------------------------------------------------------------- forward
__global__ void __launch_bounds__(kLossThreads) loss_prep_kernel(const float* __restrict__ targets, int G, int* __restrict__ nlabel) {
  __shared__ int part[kLossThreads / 32];
  const int b = blockIdx.x;
  int n = 0;
  for (int g = threadIdx.x; g < G; g += blockDim.x) {
    const float* r = targets + ((size_t)b * G + g) * 5;
    n += ((((r[0] + r[1]) + r[2]) + r[3]) + r[4]) > 0.0f;
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = n;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int w = 0; w < kLossThreads / 32; ++w) t += part[w];
    nlabel[b] = t;
  }
}

__global__ void __launch_bounds__(kLossThreads) loss_anchor_kernel(LossLevels L, const float* __restrict__ targets, const int* __restrict__ nlabel,
                                                                   float4* __restrict__ box, float2* __restrict__ sc, uint8_t* __restrict__ flag) {
  extern __shared__ float4 gts[];
  const int b = blockIdx.y, n = nlabel[b];
  for (int g = threadIdx.x; g < n; g += blockDim.x) {
    int cls;
    gts[g] = load_gt(targets, b, g, L.G, &cls);
  }
  __syncthreads();
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= L.A) return;
  const Anchor an = anchor_at(L, b, a);
  const float so = sigmoidf(an.p[4 * an.hw]);
  float S = 0.0f;
  for (int c = 0; c < L.nc; ++c) S += bce0(sqrtf(sigmoidf(an.p[(5 + c) * an.hw]) * so));
  const float xc = an.x * an.s + 0.5f * an.s, yc = an.y * an.s + 0.5f * an.s;
  bool cand = false;
  for (int g = 0; g < n && !cand; ++g) cand = in_box(gts[g], xc, yc) || in_center(gts[g], xc, yc, an.s);
  const size_t idx = (size_t)b * L.A + a;
  box[idx] = decode(an);
  sc[idx] = make_float2(S, so);
  flag[idx] = cand;
}

__global__ void __launch_bounds__(1024) loss_compact_kernel(const uint8_t* __restrict__ flag, int A, int* __restrict__ cand, int* __restrict__ ncand) {
  __shared__ int warp_tot[32];
  __shared__ int base;
  const int b = blockIdx.x, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (threadIdx.x == 0) base = 0;
  __syncthreads();
  for (int a0 = 0; a0 < A; a0 += 1024) {
    const int a = a0 + threadIdx.x;
    const bool f = a < A && flag[(size_t)b * A + a];
    const unsigned m = __ballot_sync(0xffffffffu, f);
    if (lane == 0) warp_tot[wid] = __popc(m);
    __syncthreads();
    if (wid == 0) {
      const int v = warp_tot[lane];
      int incl = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
      }
      warp_tot[lane] = incl - v;  // exclusive prefix
    }
    __syncthreads();
    if (f) cand[(size_t)b * A + base + warp_tot[wid] + __popc(m & ((1u << lane) - 1u))] = a;
    __syncthreads();
    if (threadIdx.x == 1023) base += warp_tot[31] + __popc(m);
    __syncthreads();
  }
  if (threadIdx.x == 0) ncand[b] = base;
}

// (key, index) order of the selections: smaller key first, then smaller index
__device__ __forceinline__ bool before(float k1, int i1, float k2, int i2) { return k1 < k2 || (k1 == k2 && i1 < i2); }

// Block-wide best (key, index) under `before` (largest = false) or its mirror for the largest keys; every thread gets the result.
template <bool LARGEST>
__device__ __forceinline__ void block_best(float& k, int& i, float2* red) {
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const float k2 = __shfl_xor_sync(0xffffffffu, k, o);
    const int i2 = __shfl_xor_sync(0xffffffffu, i, o);
    if (LARGEST ? before(-k2, i2, -k, i) : before(k2, i2, k, i)) { k = k2; i = i2; }
  }
  __syncthreads();  // (red is reused by consecutive rounds)
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = make_float2(k, __int_as_float(i));
  __syncthreads();
  k = red[0].x;
  i = __float_as_int(red[0].y);
  for (int w = 1; w < kLossThreads / 32; ++w) {
    const float k2 = red[w].x;
    const int i2 = __float_as_int(red[w].y);
    if (LARGEST ? before(-k2, i2, -k, i) : before(k2, i2, k, i)) { k = k2; i = i2; }
  }
}

__global__ void __launch_bounds__(kLossThreads) loss_gt_kernel(LossLevels L, const float* __restrict__ targets, const int* __restrict__ nlabel,
                                                               const int* __restrict__ cand, const int* __restrict__ ncand, const float4* __restrict__ box,
                                                               const float2* __restrict__ sc, int* __restrict__ cnt, int* __restrict__ taker) {
  __shared__ float2 red[kLossThreads / 32];
  const int g = blockIdx.x, b = blockIdx.y;
  if (g >= nlabel[b]) return;
  const int n = ncand[b];
  if (n == 0) return;  // no candidate anchor in the image: the GT gets no match (the reference's topk raises here)
  int cls;
  const float4 gt = load_gt(targets, b, g, L.G, &cls);
  // per-thread top-10 IoUs (descending; -1 = empty) and 10 lowest (cost, anchor) (ascending; (FLT_MAX, INT_MAX) = empty), in registers
  float ti[kTopK], ck[kTopK];
  int ci[kTopK];
#pragma unroll
  for (int t = 0; t < kTopK; ++t) { ti[t] = -1.0f; ck[t] = FLT_MAX; ci[t] = INT_MAX; }
  for (int j = threadIdx.x; j < n; j += blockDim.x) {
    const int a = cand[(size_t)b * L.A + j];
    const Anchor an = anchor_at(L, b, a);
    float iou;
    const float c = cost(L, an, load_cost(box, sc, (size_t)b * L.A + a), gt, cls, &iou);
    if (iou > ti[kTopK - 1]) {
      ti[kTopK - 1] = iou;
#pragma unroll
      for (int t = kTopK - 1; t > 0; --t)
        if (ti[t] > ti[t - 1]) { const float v = ti[t]; ti[t] = ti[t - 1]; ti[t - 1] = v; }
    }
    if (before(c, a, ck[kTopK - 1], ci[kTopK - 1])) {
      ck[kTopK - 1] = c;
      ci[kTopK - 1] = a;
#pragma unroll
      for (int t = kTopK - 1; t > 0; --t)
        if (before(ck[t], ci[t], ck[t - 1], ci[t - 1])) {
          const float v = ck[t]; ck[t] = ck[t - 1]; ck[t - 1] = v;
          const int u = ci[t]; ci[t] = ci[t - 1]; ci[t - 1] = u;
        }
    }
  }
  // dynamic k = max(1, int(sum of the top min(10, n) IoUs)), summed in descending order
  float sum = 0.0f;
  for (int r = 0; r < kTopK; ++r) {
    float k = ti[0];
    int i = threadIdx.x;
    block_best<true>(k, i, red);
    if (k < 0.0f) break;
    sum += k;
    if (i == (int)threadIdx.x) {
#pragma unroll
      for (int t = 0; t < kTopK - 1; ++t) ti[t] = ti[t + 1];
      ti[kTopK - 1] = -1.0f;
    }
  }
  const int dk = max(1, (int)sum);
  for (int r = 0; r < dk; ++r) {
    float k = ck[0];
    int i = ci[0];
    block_best<false>(k, i, red);
    if (i == INT_MAX) break;
    if (i == ci[0]) {  // the owner of the winning anchor records the match and pops it
      atomicAdd(cnt + (size_t)b * L.A + i, 1);
      taker[(size_t)b * L.A + i] = g;  // (read only where exactly one GT took the anchor)
#pragma unroll
      for (int t = 0; t < kTopK - 1; ++t) { ck[t] = ck[t + 1]; ci[t] = ci[t + 1]; }
      ck[kTopK - 1] = FLT_MAX;
      ci[kTopK - 1] = INT_MAX;
    }
  }
}

// IOUloss (yolox_loss.py:34-69, loss_type "iou"): iou with +1e-16 in the denominator
__device__ __forceinline__ float loss_iou(float4 p, float4 t) {
  const float tlx = fmaxf(p.x - p.z / 2.0f, t.x - t.z / 2.0f), tly = fmaxf(p.y - p.w / 2.0f, t.y - t.w / 2.0f);
  const float brx = fminf(p.x + p.z / 2.0f, t.x + t.z / 2.0f), bry = fminf(p.y + p.w / 2.0f, t.y + t.w / 2.0f);
  const float area_p = p.z * p.w, area_g = t.z * t.w;
  const float en = (tlx < brx && tly < bry) ? 1.0f : 0.0f;
  const float area_i = (brx - tlx) * (bry - tly) * en;
  return area_i / (area_p + area_g - area_i + 1e-16f);
}


// d(1 - iou^2) / d(pred (x, y, w, h)) of loss_iou, as torch.autograd differentiates IOUloss (torch.max / torch.min split the gradient
// evenly between equal operands; the enable factor is a constant)
__device__ __forceinline__ float4 loss_iou_grad(float4 p, float4 t) {
  const float ax = p.x - p.z / 2.0f, bx = t.x - t.z / 2.0f, ay = p.y - p.w / 2.0f, by = t.y - t.w / 2.0f;
  const float cx = p.x + p.z / 2.0f, dx = t.x + t.z / 2.0f, cy = p.y + p.w / 2.0f, dy = t.y + t.w / 2.0f;
  const float tlx = fmaxf(ax, bx), tly = fmaxf(ay, by), brx = fminf(cx, dx), bry = fminf(cy, dy);
  const float wtx = ax > bx ? 1.0f : (ax == bx ? 0.5f : 0.0f), wty = ay > by ? 1.0f : (ay == by ? 0.5f : 0.0f);
  const float wbx = cx < dx ? 1.0f : (cx == dx ? 0.5f : 0.0f), wby = cy < dy ? 1.0f : (cy == dy ? 0.5f : 0.0f);
  const float en = (tlx < brx && tly < bry) ? 1.0f : 0.0f;
  const float hx = brx - tlx, hy = bry - tly;
  const float area_i = hx * hy * en, area_p = p.z * p.w, area_g = t.z * t.w;
  const float U = area_p + area_g - area_i + 1e-16f;
  const float iou = area_i / U;
  const float d_iou = -2.0f * iou;
  const float dI = d_iou * (1.0f / U + area_i / (U * U));  // d loss / d area_i
  const float dP = d_iou * (-area_i / (U * U));            // d loss / d area_p
  const float d_tlx = -hy * en * dI, d_brx = hy * en * dI, d_tly = -hx * en * dI, d_bry = hx * en * dI;
  return make_float4(d_tlx * wtx + d_brx * wbx, d_tly * wty + d_bry * wby,
                     -0.5f * d_tlx * wtx + 0.5f * d_brx * wbx + dP * p.w, -0.5f * d_tly * wty + 0.5f * d_bry * wby + dP * p.z);
}

__global__ void __launch_bounds__(kLossThreads) loss_resolve_kernel(LossLevels L, int B, const float* __restrict__ targets, const int* __restrict__ nlabel,
                                                                    const float4* __restrict__ box, const float2* __restrict__ sc, const int* __restrict__ cnt,
                                                                    const int* __restrict__ taker, int* __restrict__ matched_gt, float* __restrict__ matched_iou,
                                                                    double* __restrict__ partial) {
  __shared__ double red[kLossThreads / 32][4];
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  double v[4] = {0.0, 0.0, 0.0, 0.0};  // sum of (1 - iou^2), objectness BCE, class BCE, foreground count
  if (idx < (long long)B * L.A) {
    const int b = (int)(idx / L.A), a = (int)(idx % L.A);
    const Anchor an = anchor_at(L, b, a);
    const int c = cnt[idx];
    int m = -1;
    if (c == 1) {
      m = taker[idx];
    } else if (c > 1) {  // taken by several GTs: the argmin of the cost over all GTs, the lower GT index on ties
      const AnchorCost ac = load_cost(box, sc, idx);
      float best = 0.0f;
      for (int g = 0; g < nlabel[b]; ++g) {
        int cls;
        const float4 gt = load_gt(targets, b, g, L.G, &cls);
        float iou;
        const float cg = cost(L, an, ac, gt, cls, &iou);
        if (m < 0 || cg < best) { best = cg; m = g; }
      }
    }
    v[1] = bce_logits(an.p[4 * an.hw], m >= 0 ? 1.0f : 0.0f);
    float miou = 0.0f;
    if (m >= 0) {
      int cls;
      const float4 gt = load_gt(targets, b, m, L.G, &cls);
      const float4 pb = box[idx];
      miou = pair_iou(gt, pb);
      const float li = loss_iou(pb, gt);
      v[0] = 1.0f - li * li;
      for (int k = 0; k < L.nc; ++k) v[2] += bce_logits(an.p[(5 + k) * an.hw], k == cls ? miou : 0.0f);
      v[3] = 1.0;
    }
    matched_gt[idx] = m;
    matched_iou[idx] = miou;
  }
  block_sum<kLossThreads>(v, red);
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < 4; ++k) partial[(size_t)blockIdx.x * 4 + k] = v[k];
  }
}

__global__ void __launch_bounds__(kLossThreads) loss_final_kernel(const double* __restrict__ partial, int nblk, const int* __restrict__ nlabel, int B,
                                                                  float* __restrict__ out) {
  __shared__ double red[4][kLossThreads];
  double v[4] = {0.0, 0.0, 0.0, 0.0};
  for (int i = threadIdx.x; i < nblk; i += blockDim.x) {
#pragma unroll
    for (int k = 0; k < 4; ++k) v[k] += partial[(size_t)i * 4 + k];
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) red[k][threadIdx.x] = v[k];
  __syncthreads();
  for (int s = kLossThreads / 2; s; s >>= 1) {
    if ((int)threadIdx.x < s) {
#pragma unroll
      for (int k = 0; k < 4; ++k) red[k][threadIdx.x] += red[k][threadIdx.x + s];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    long long ngt = 0;
    for (int b = 0; b < B; ++b) ngt += nlabel[b];
    const double nfg = fmax(red[3][0], 1.0);  // num_fg = max(sum of the images' foreground counts, 1)
    const float li = (float)(red[0][0] / nfg), lo = (float)(red[1][0] / nfg), lc = (float)(red[2][0] / nfg);
    out[0] = (5.0f * li + lo) + lc;
    out[1] = 5.0f * li;
    out[2] = lo;
    out[3] = lc;
    out[4] = (float)(nfg / (double)(ngt > 1 ? ngt : 1));
    out[5] = (float)nfg;
  }
}

// --------------------------------------------------------------------------------------------------------------------------- backward
__global__ void __launch_bounds__(kLossThreads) loss_bwd_kernel(LossLevels L, const float* __restrict__ targets, const int* __restrict__ matched_gt,
                                                                const float* __restrict__ matched_iou, const float* __restrict__ fwd_out,
                                                                const float* __restrict__ gout) {
  const int b = blockIdx.y, a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= L.A) return;
  const Anchor an = anchor_at(L, b, a);
  const size_t idx = (size_t)b * L.A + a;
  const float nf = fwd_out[5];
  // loss = iou_loss + conf_loss + cls_loss, each also an output of its own: d/d(term) = g_loss + g_term
  const float cI = 5.0f * (gout[0] + gout[1]) / nf, cO = (gout[0] + gout[2]) / nf, cC = (gout[0] + gout[3]) / nf;
  const int m = matched_gt[idx];
  const int hw = an.hw;
  an.g[4 * hw] = (sigmoidf(an.p[4 * hw]) - (m >= 0 ? 1.0f : 0.0f)) * cO;
  if (m >= 0) {
    int cls;
    const float4 gt = load_gt(targets, b, m, L.G, &cls);
    const float4 pb = decode(an);
    const float4 d = loss_iou_grad(pb, gt);
    an.g[0] = d.x * an.s * cI;
    an.g[hw] = d.y * an.s * cI;
    an.g[2 * hw] = d.z * pb.z * cI;  // d(exp(p) s) / dp = exp(p) s
    an.g[3 * hw] = d.w * pb.w * cI;
    const float miou = matched_iou[idx];
    for (int k = 0; k < L.nc; ++k) an.g[(5 + k) * hw] = (sigmoidf(an.p[(5 + k) * hw]) - (k == cls ? miou : 0.0f)) * cC;
  } else {
#pragma unroll
    for (int k = 0; k < 4; ++k) an.g[k * hw] = 0.0f;
    for (int k = 0; k < L.nc; ++k) an.g[(5 + k) * hw] = 0.0f;
  }
}

// --------------------------------------------------------------------------------------------------------------------------- host
struct LossWs {
  float4* box;
  float2* sc;
  uint8_t* flag;
  int *cand, *cnt, *taker, *nlabel, *ncand;
  double* partial;
  size_t bytes;
};

inline int resolve_blocks(int B, int A) { return (int)(((long long)B * A + kLossThreads - 1) / kLossThreads); }

LossWs loss_ws(void* base, int B, int A) {
  WsCarver c(base);
  LossWs w{};
  const size_t n = (size_t)B * A;
  w.box = static_cast<float4*>(c.take(n * sizeof(float4)));
  w.sc = static_cast<float2*>(c.take(n * sizeof(float2)));
  w.flag = static_cast<uint8_t*>(c.take(n));
  w.cand = static_cast<int*>(c.take(n * 4));
  w.cnt = static_cast<int*>(c.take(n * 4));
  w.taker = static_cast<int*>(c.take(n * 4));
  w.nlabel = static_cast<int*>(c.take((size_t)B * 4));
  w.ncand = static_cast<int*>(c.take((size_t)B * 4));
  w.partial = static_cast<double*>(c.take((size_t)resolve_blocks(B, A) * 4 * sizeof(double)));
  w.bytes = c.bytes();
  return w;
}

// Validates the level description shared by the forward and the backward and fills L (gradients: grads, may be NULL in the forward).
int make_levels(const char* what, const float* const* preds, const int32_t* shapes, const float* strides, int32_t nlev, int32_t nc, int32_t B,
                int32_t max_gt, const float* targets, float* const* grads, LossLevels* L) {
  CVB_REQUIRE(preds && shapes && strides && targets, "%s: preds, shapes, strides and targets are required", what);
  CVB_REQUIRE(nlev >= 1 && nlev <= kLossMaxLevels, "%s: 1 to %d levels supported (got %d)", what, kLossMaxLevels, nlev);
  CVB_REQUIRE(nc >= 1, "%s: num_classes must be >= 1 (got %d)", what, nc);
  CVB_REQUIRE(B >= 1, "%s: batch must be >= 1 (got %d)", what, B);
  CVB_REQUIRE(max_gt >= 1 && max_gt <= kLossMaxGt, "%s: max_gt must be in [1, %d] GT rows per image (got %d)", what, kLossMaxGt, max_gt);
  CVB_REQUIRE(is_aligned(targets, 4), "%s: targets must be 4-byte aligned", what);
  *L = LossLevels{};
  long long A = 0;
  for (int l = 0; l < nlev; ++l) {
    const int32_t* s = shapes + 4 * l;
    CVB_REQUIRE(preds[l] && is_aligned(preds[l], 4), "%s: level %d output missing or not 4-byte aligned", what, l);
    CVB_REQUIRE(s[0] == B && s[1] == 5 + nc && s[2] > 0 && s[3] > 0,
                "%s: level %d output must be [B=%d, 5 + num_classes=%d, h > 0, w > 0] (got [%d, %d, %d, %d])", what, l, B, 5 + nc, s[0], s[1], s[2], s[3]);
    CVB_REQUIRE(strides[l] > 0.0f, "%s: level %d stride must be > 0 (got %g)", what, l, (double)strides[l]);
    if (grads) CVB_REQUIRE(grads[l] && is_aligned(grads[l], 4), "%s: level %d gradient missing or not 4-byte aligned", what, l);
    L->p[l] = preds[l];
    L->g[l] = grads ? grads[l] : nullptr;
    L->h[l] = s[2];
    L->w[l] = s[3];
    L->s[l] = strides[l];
    L->off[l] = (int)A;
    A += (long long)s[2] * s[3];
    CVB_REQUIRE((long long)B * (5 + nc) * s[2] * s[3] < (1LL << 40), "%s: level %d too large", what, l);
  }
  CVB_REQUIRE((long long)B * A < INT_MAX, "%s: B x anchors too large (%lld)", what, (long long)B * A);
  L->off[nlev] = (int)A;
  L->nlev = nlev;
  L->A = (int)A;
  L->nc = nc;
  L->G = max_gt;
  return CVB_OK;
}

}  // namespace
}  // namespace cvb

using namespace cvb;

extern "C" size_t cvb_train_yolox_loss_workspace_bytes(int32_t B, int32_t A) {
  if (B <= 0 || A <= 0) return 0;
  return loss_ws(nullptr, B, A).bytes;
}

extern "C" int cvb_train_yolox_loss_fwd(const float* const* preds, const int32_t* shapes, const float* strides, int32_t nlev, int32_t nc, const float* targets,
                                        int32_t B, int32_t max_gt, int32_t* matched_gt, float* matched_iou, float* out, void* workspace, size_t ws_bytes,
                                        void* stream) {
  LossLevels L;
  const int rc = make_levels("train_yolox_loss_fwd", preds, shapes, strides, nlev, nc, B, max_gt, targets, nullptr, &L);
  if (rc != CVB_OK) return rc;
  CVB_REQUIRE(matched_gt && matched_iou && out && is_aligned(matched_gt, 4) && is_aligned(matched_iou, 4) && is_aligned(out, 4),
              "train_yolox_loss_fwd: matched_gt, matched_iou and out are required, 4-byte aligned");
  const LossWs w = loss_ws(workspace, B, L.A);
  CVB_REQUIRE(workspace && is_aligned(workspace, 256), "train_yolox_loss_fwd: workspace required, 256-byte aligned");
  CVB_REQUIRE(ws_bytes >= w.bytes, "train_yolox_loss_fwd: workspace of %zu bytes too small (%zu needed)", ws_bytes, w.bytes);
  cudaStream_t st = as_stream(stream);
  CVB_CHECK_CUDA(cudaMemsetAsync(w.cnt, 0, (size_t)B * L.A * sizeof(int), st));
  loss_prep_kernel<<<B, kLossThreads, 0, st>>>(targets, max_gt, w.nlabel);
  loss_anchor_kernel<<<dim3(ceil_div(L.A, kLossThreads), B), kLossThreads, (size_t)max_gt * sizeof(float4), st>>>(L, targets, w.nlabel, w.box, w.sc, w.flag);
  loss_compact_kernel<<<B, 1024, 0, st>>>(w.flag, L.A, w.cand, w.ncand);
  loss_gt_kernel<<<dim3(max_gt, B), kLossThreads, 0, st>>>(L, targets, w.nlabel, w.cand, w.ncand, w.box, w.sc, w.cnt, w.taker);
  const int nblk = resolve_blocks(B, L.A);
  loss_resolve_kernel<<<nblk, kLossThreads, 0, st>>>(L, B, targets, w.nlabel, w.box, w.sc, w.cnt, w.taker, matched_gt, matched_iou, w.partial);
  loss_final_kernel<<<1, kLossThreads, 0, st>>>(w.partial, nblk, w.nlabel, B, out);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch(6);
  return CVB_OK;
}

extern "C" int cvb_train_yolox_loss_bwd(const float* const* preds, const int32_t* shapes, const float* strides, int32_t nlev, int32_t nc, const float* targets,
                                        int32_t B, int32_t max_gt, const int32_t* matched_gt, const float* matched_iou, const float* fwd_out,
                                        const float* grad_out, float* const* grads, void* stream) {
  CVB_REQUIRE(grads, "train_yolox_loss_bwd: grads required");
  LossLevels L;
  const int rc = make_levels("train_yolox_loss_bwd", preds, shapes, strides, nlev, nc, B, max_gt, targets, grads, &L);
  if (rc != CVB_OK) return rc;
  CVB_REQUIRE(matched_gt && matched_iou && fwd_out && grad_out && is_aligned(matched_gt, 4) && is_aligned(matched_iou, 4) &&
                  is_aligned(fwd_out, 4) && is_aligned(grad_out, 4),
              "train_yolox_loss_bwd: matched_gt, matched_iou, fwd_out and grad_out are required, 4-byte aligned");
  loss_bwd_kernel<<<dim3(ceil_div(L.A, kLossThreads), B), kLossThreads, 0, as_stream(stream)>>>(L, targets, matched_gt, matched_iou, fwd_out, grad_out);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}
