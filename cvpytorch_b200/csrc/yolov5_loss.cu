// The YOLOv5 training loss on the device: target-to-anchor matching (build_targets), the CIoU box / IoU-target objectness / class BCE
// losses and their gradient with respect to the detect convs' fp32 NCHW outputs (src/losses/yolov5_loss.py:135-278; restated in
// oracle/yolov5_train_oracle.py).  A level's output [B, na * (5 + nc), ny, nx] is read in place as [B, na, 5 + nc, ny, nx].
//
// Forward (cvb_train_yolov5_loss_fwd), stream-ordered, no host sync, CUDA-graph capturable (every buffer is sized on the host from nt):
//   1. v5_cand_kernel   one CTA per level: the candidate list in the reference's order (offset-major: centre, +x, +y, -x, -y; then anchor;
//                       then target), compacted with a block scan, with the clamped cell, tbox = gxy - clamped cell, the anchor and the class.
//   2. v5_rank_kernel   the stable sort of the candidates by cell: rank = #(cell, index) pairs before the candidate's (exact, no atomics).
//   3. v5_term_kernel   one thread per candidate: CIoU of the decoded prediction, 1 - CIoU and the class BCE sum.
//   4. v5_seg_kernel    one thread per sorted position; the first of each cell's run takes the last candidate in candidate order (last write
//                       wins, as the reference's index_put_ does while it runs serially) for tobj = (1 - gr) + gr * clamp(CIoU, 0), and the objectness
//                       correction BCE(x, tobj) - BCE(x, 0) of that cell.
//   5. v5_obj_kernel    every objectness logit: BCE(x, 0), summed per CTA (block_sum).
//   6. v5_final_kernel  one CTA: the per-level means from fp64 sums (block_sum) -> loss, lbox, lobj, lcls.
// Backward (cvb_train_yolov5_loss_bwd): v5_fill_kernel writes every gradient element (objectness d/dx of BCE(x, 0), zeros elsewhere);
// v5_cell_grad_kernel then rewrites the channels of each candidate cell, summing its candidates' box and class gradients in candidate
// order.  No float atomics: the loss and the gradient are bitwise reproducible.
//
// Precision: fp32 in the reference's operation order (compiled with --fmad=false), sums in fp64.
#include <limits.h>

#include <algorithm>

#include "internal.h"

namespace cvb {
namespace {

constexpr int kV5MaxLevels = 4;
constexpr int kV5MaxAnchors = 8;
constexpr int kV5Threads = 256;
constexpr int kV5ObjBlocks = 128;  // CTAs per level of the objectness pass (a fixed grid: a fixed summation tree)

struct V5Levels {
  const float* p[kV5MaxLevels];  // [B, na, 5 + nc, ny, nx] fp32
  float* g[kV5MaxLevels];        // gradients, same shapes (backward only)
  int ny[kV5MaxLevels], nx[kV5MaxLevels];
  float anchor[kV5MaxLevels][kV5MaxAnchors][2];  // grid units
  float balance[kV5MaxLevels];
  int nlev, na, nc, B, nt, cap;
  float anchor_t, hyp_box, hyp_obj, hyp_cls, gr;
};

struct Cand {   // cand_idx row
  int b, a, gj, gi, cls;
};

__device__ __forceinline__ size_t cell_base(const V5Levels& L, int l, int b, int a, int gj, int gi) {
  const int no = 5 + L.nc;
  return (((size_t)b * L.na + a) * no * L.ny[l] + gj) * L.nx[l] + gi;  // channel c at + c * ny * nx
}

// --------------------------------------------------------------------------------------------------------------------------- forward
// Slot s = (o * na + a) * nt + t; the slots of a level are scanned in order and the valid ones compacted, so the list is the reference's.
__global__ void __launch_bounds__(1024) v5_cand_kernel(V5Levels L, const float* __restrict__ targets, int* __restrict__ cand_idx, float* __restrict__ cand_box,
                                                       int* __restrict__ ncand, int* __restrict__ key) {
  __shared__ int warp_tot[32];
  __shared__ int base;
  const int l = blockIdx.x, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int nx = L.nx[l], ny = L.ny[l];
  const float fx = (float)nx, fy = (float)ny;
  const int slots = 5 * L.na * L.nt;
  if (threadIdx.x == 0) base = 0;
  __syncthreads();
  for (int s0 = 0; s0 < slots; s0 += 1024) {
    const int s = s0 + threadIdx.x;
    bool ok = false;
    Cand c{};
    float tb[6];
    if (s < slots) {
      const int o = s / (L.na * L.nt), r = s % (L.na * L.nt), a = r / L.nt, t = r % L.nt;
      const float* row = targets + (size_t)t * 6;
      const float gx = row[2] * fx, gy = row[3] * fy, gw = row[4] * fx, gh = row[5] * fy;
      const float aw = L.anchor[l][a][0], ah = L.anchor[l][a][1];
      const float rw = gw / aw, rh = gh / ah;
      const float mw = fmaxf(rw, 1.0f / rw), mh = fmaxf(rh, 1.0f / rh);
      ok = fmaxf(mw, mh) < L.anchor_t;  // (both fp32 compares of the reference: max(r, 1 / r).max(2) < anchor_t)
      const float ix = fx - gx, iy = fy - gy;
      const float g = 0.5f;
      float ox = 0.0f, oy = 0.0f;
      if (o == 1) { ok = ok && fmodf(gx, 1.0f) < g && gx > 1.0f; ox = g; }
      if (o == 2) { ok = ok && fmodf(gy, 1.0f) < g && gy > 1.0f; oy = g; }
      if (o == 3) { ok = ok && fmodf(ix, 1.0f) < g && ix > 1.0f; ox = -g; }
      if (o == 4) { ok = ok && fmodf(iy, 1.0f) < g && iy > 1.0f; oy = -g; }
      c.b = (int)row[0];
      c.cls = (int)row[1];
      ok = ok && c.b >= 0 && c.b < L.B;  // (an image index outside the batch matches nothing)
      c.a = a;
      c.gi = min(max((int)(gx - ox), 0), nx - 1);  // (truncation toward zero, as .long(); then the in-place clamp)
      c.gj = min(max((int)(gy - oy), 0), ny - 1);
      tb[0] = gx - (float)c.gi;                    // tbox uses the clamped cell
      tb[1] = gy - (float)c.gj;
      tb[2] = gw;
      tb[3] = gh;
      tb[4] = aw;
      tb[5] = ah;
    }
    const unsigned m = __ballot_sync(0xffffffffu, ok);
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
      warp_tot[lane] = incl - v;
    }
    __syncthreads();
    if (ok) {
      const size_t k = (size_t)l * L.cap + base + warp_tot[wid] + __popc(m & ((1u << lane) - 1u));
      int* ci = cand_idx + k * 5;
      ci[0] = c.b; ci[1] = c.a; ci[2] = c.gj; ci[3] = c.gi; ci[4] = c.cls;
#pragma unroll
      for (int i = 0; i < 6; ++i) cand_box[k * 6 + i] = tb[i];
      key[k] = ((c.b * L.na + c.a) * ny + c.gj) * nx + c.gi;
    }
    __syncthreads();
    if (threadIdx.x == 1023) base += warp_tot[31] + __popc(m);
    __syncthreads();
  }
  if (threadIdx.x == 0) ncand[l] = base;
}

// sorted[rank] = k with rank = #{j : (key_j, j) < (key_k, k)}: a stable sort by cell, exact and without atomics.
__global__ void __launch_bounds__(kV5Threads) v5_rank_kernel(int cap, const int* __restrict__ key, const int* __restrict__ ncand, int* __restrict__ sorted) {
  __shared__ int tk[kV5Threads];
  const int l = blockIdx.y, n = ncand[l];
  if ((int)blockIdx.x * kV5Threads >= n) return;
  const int k = blockIdx.x * kV5Threads + threadIdx.x;
  const int* kl = key + (size_t)l * cap;
  const int mk = k < n ? kl[k] : 0;
  int rank = 0;
  for (int j0 = 0; j0 < n; j0 += kV5Threads) {
    const int j = j0 + threadIdx.x;
    tk[threadIdx.x] = j < n ? kl[j] : INT_MAX;
    __syncthreads();
    const int m = min(kV5Threads, n - j0);
    for (int jj = 0; jj < m; ++jj) {
      const int kj = tk[jj];
      rank += (kj < mk) || (kj == mk && j0 + jj < k);
    }
    __syncthreads();
  }
  if (k < n) sorted[(size_t)l * cap + rank] = k;
}

// The decoded prediction of candidate k: pxy = 2 sigmoid - 0.5, pwh = (2 sigmoid)^2 anchor (yolov5_loss.py:161-163)
struct Pred {
  float sx, sy, sw, sh;  // sigmoids
  float px, py, pw, ph;
};

__device__ __forceinline__ Pred decode(const float* base, size_t hw, const float* tb) {
  Pred p;
  p.sx = sigmoidf(base[0]);
  p.sy = sigmoidf(base[hw]);
  p.sw = sigmoidf(base[2 * hw]);
  p.sh = sigmoidf(base[3 * hw]);
  p.px = p.sx * 2.0f - 0.5f;
  p.py = p.sy * 2.0f - 0.5f;
  const float tw = p.sw * 2.0f, th = p.sh * 2.0f;
  p.pw = (tw * tw) * tb[4];
  p.ph = (th * th) * tb[5];
  return p;
}

constexpr float kEps = 1e-7f;
constexpr float kV = 0.40528473456935108578f;  // 4 / pi^2

// bbox_iou(pbox, tbox, x1y1x2y2=False, CIoU=True) (yolov5_loss.py:11-52) with the reference's eps placement.  With grad != nullptr:
// d(ciou)/d(px, py, pw, ph) as torch.autograd gives it (alpha detached; min / max split the gradient in half at equality; clamp(0) passes
// it at 0).
__device__ __forceinline__ float ciou(float px, float py, float pw, float ph, const float* tb, float* grad) {
  const float b1x1 = px - pw / 2.0f, b1x2 = px + pw / 2.0f, b1y1 = py - ph / 2.0f, b1y2 = py + ph / 2.0f;
  const float b2x1 = tb[0] - tb[2] / 2.0f, b2x2 = tb[0] + tb[2] / 2.0f, b2y1 = tb[1] - tb[3] / 2.0f, b2y2 = tb[1] + tb[3] / 2.0f;
  const float iw = fminf(b1x2, b2x2) - fmaxf(b1x1, b2x1), ih = fminf(b1y2, b2y2) - fmaxf(b1y1, b2y1);
  const float iwc = fmaxf(iw, 0.0f), ihc = fmaxf(ih, 0.0f);
  const float inter = iwc * ihc;
  const float w1 = b1x2 - b1x1, h1 = b1y2 - b1y1 + kEps;
  const float w2 = b2x2 - b2x1, h2 = b2y2 - b2y1 + kEps;
  const float uni = w1 * h1 + w2 * h2 - inter + kEps;
  const float iou = inter / uni;
  const float cw = fmaxf(b1x2, b2x2) - fminf(b1x1, b2x1), ch = fmaxf(b1y2, b2y2) - fminf(b1y1, b2y1);
  const float c2 = cw * cw + ch * ch + kEps;
  const float dx = b2x1 + b2x2 - b1x1 - b1x2, dy = b2y1 + b2y2 - b1y1 - b1y2;
  const float rho2 = (dx * dx + dy * dy) / 4.0f;
  const float at = atanf(w2 / h2) - atanf(w1 / h1);
  const float v = kV * (at * at);
  const float alpha = v / (v - iou + (1.0f + kEps));
  const float out = iou - (rho2 / c2 + v * alpha);
  if (grad) {
    // d(out) = 1 * d(iou) - d(rho2) / c2 + rho2 / c2^2 d(c2) - alpha d(v)
    const float g_rho2 = -1.0f / c2, g_c2 = rho2 / (c2 * c2), g_v = -alpha;
    const float g_at = g_v * kV * (2.0f * at);
    const float u = w1 / h1, g_u = -g_at / (1.0f + u * u);
    float g_w1 = g_u / h1, g_h1 = -g_u * w1 / (h1 * h1);
    const float g_inter0 = 1.0f / uni, g_uni = -inter / (uni * uni);
    g_w1 += g_uni * h1;
    g_h1 += g_uni * w1;
    const float g_inter = g_inter0 - g_uni;
    const float g_iw = iw >= 0.0f ? g_inter * ihc : 0.0f, g_ih = ih >= 0.0f ? g_inter * iwc : 0.0f;
    // share of a min / max operand: 1 if it is the selected one, 0.5 on a tie
    auto lo = [](float a, float b) { return a < b ? 1.0f : (a == b ? 0.5f : 0.0f); };
    auto hi = [](float a, float b) { return a > b ? 1.0f : (a == b ? 0.5f : 0.0f); };
    const float g_cw = g_c2 * (2.0f * cw), g_ch = g_c2 * (2.0f * ch);
    const float g_dx = g_rho2 / 4.0f * (2.0f * dx), g_dy = g_rho2 / 4.0f * (2.0f * dy);
    const float g_x2 = g_iw * lo(b1x2, b2x2) + g_cw * hi(b1x2, b2x2) - g_dx + g_w1;
    const float g_x1 = -g_iw * hi(b1x1, b2x1) - g_cw * lo(b1x1, b2x1) - g_dx - g_w1;
    const float g_y2 = g_ih * lo(b1y2, b2y2) + g_ch * hi(b1y2, b2y2) - g_dy + g_h1;
    const float g_y1 = -g_ih * hi(b1y1, b2y1) - g_ch * lo(b1y1, b2y1) - g_dy - g_h1;
    grad[0] = g_x1 + g_x2;
    grad[1] = g_y1 + g_y2;
    grad[2] = (g_x2 - g_x1) / 2.0f;
    grad[3] = (g_y2 - g_y1) / 2.0f;
  }
  return out;
}

__global__ void __launch_bounds__(kV5Threads) v5_term_kernel(V5Levels L, const int* __restrict__ cand_idx, const float* __restrict__ cand_box,
                                                             const int* __restrict__ ncand, float* __restrict__ score, double* __restrict__ term) {
  const int l = blockIdx.y, k = blockIdx.x * kV5Threads + threadIdx.x;
  if (k >= ncand[l]) return;
  const size_t i = (size_t)l * L.cap + k;
  const int* ci = cand_idx + i * 5;
  const float* tb = cand_box + i * 6;
  const size_t hw = (size_t)L.ny[l] * L.nx[l];
  const float* base = L.p[l] + cell_base(L, l, ci[0], ci[1], ci[2], ci[3]);
  const Pred p = decode(base, hw, tb);
  const float c = ciou(p.px, p.py, p.pw, p.ph, tb, nullptr);
  score[i] = c;
  term[2 * i] = (double)(1.0f - c);
  double cls = 0.0;
  if (L.nc > 1)
    for (int j = 0; j < L.nc; ++j) cls += (double)bce_logits(base[(5 + j) * hw], j == ci[4] ? 1.0f : 0.0f);
  term[2 * i + 1] = cls;
}

// tobj of the candidate cell whose sorted run starts at p (clamp(0) keeps a NaN, as torch's clamp does)
__device__ __forceinline__ float cell_tobj(const V5Levels& L, const float* score_l, const int* sorted_l, const int* key_l, int n, int p, int* last) {
  const int kk = key_l[sorted_l[p]];
  int q = p;
  while (q + 1 < n && key_l[sorted_l[q + 1]] == kk) ++q;
  *last = q;
  const float s = score_l[sorted_l[q]];
  return (1.0f - L.gr) + L.gr * (s < 0.0f ? 0.0f : s);
}

__device__ __forceinline__ bool run_head(const int* sorted_l, const int* key_l, int p) {
  return p == 0 || key_l[sorted_l[p - 1]] != key_l[sorted_l[p]];
}

__global__ void __launch_bounds__(kV5Threads) v5_seg_kernel(V5Levels L, const int* __restrict__ cand_idx, const int* __restrict__ ncand, const int* __restrict__ key,
                                                            const int* __restrict__ sorted, const float* __restrict__ score, double* __restrict__ corr) {
  const int l = blockIdx.y, p = blockIdx.x * kV5Threads + threadIdx.x, n = ncand[l];
  if (p >= n) return;
  const size_t off = (size_t)l * L.cap;
  double c = 0.0;
  if (run_head(sorted + off, key + off, p)) {
    int q;
    const float t = cell_tobj(L, score + off, sorted + off, key + off, n, p, &q);
    const int* ci = cand_idx + (off + sorted[off + p]) * 5;
    const float x = L.p[l][cell_base(L, l, ci[0], ci[1], ci[2], ci[3]) + 4 * (size_t)L.ny[l] * L.nx[l]];
    c = (double)bce_logits(x, t) - (double)bce_logits(x, 0.0f);
  }
  corr[off + p] = c;
}

__global__ void __launch_bounds__(kV5Threads) v5_obj_kernel(V5Levels L, double* __restrict__ partial) {
  __shared__ double red[kV5Threads / 32][1];
  const int l = blockIdx.y;
  const long long hw = (long long)L.ny[l] * L.nx[l], n = (long long)L.B * L.na * hw;
  double v[1] = {0.0};
  for (long long i = blockIdx.x * (long long)kV5Threads + threadIdx.x; i < n; i += (long long)kV5ObjBlocks * kV5Threads) {
    const long long ba = i / hw;
    v[0] += (double)bce_logits(L.p[l][(ba * (5 + L.nc) + 4) * hw + i % hw], 0.0f);
  }
  block_sum<kV5Threads>(v, red);
  if (threadIdx.x == 0) partial[l * kV5ObjBlocks + blockIdx.x] = v[0];
}

__global__ void __launch_bounds__(kV5Threads) v5_final_kernel(V5Levels L, const int* __restrict__ ncand, const double* __restrict__ term,
                                                              const double* __restrict__ corr, const double* __restrict__ partial, float* __restrict__ out) {
  __shared__ double red[kV5Threads / 32][3];
  float lbox = 0.0f, lobj = 0.0f, lcls = 0.0f;
  for (int l = 0; l < L.nlev; ++l) {
    const int n = ncand[l];
    const size_t off = (size_t)l * L.cap;
    double v[3] = {0.0, 0.0, 0.0};  // box, class, objectness
    for (int k = threadIdx.x; k < n; k += kV5Threads) {
      v[0] += term[2 * (off + k)];
      v[1] += term[2 * (off + k) + 1];
      v[2] += corr[off + k];
    }
    for (int j = threadIdx.x; j < kV5ObjBlocks; j += kV5Threads) v[2] += partial[l * kV5ObjBlocks + j];
    block_sum<kV5Threads>(v, red);
    if (n > 0) {
      lbox += (float)(v[0] / n);
      if (L.nc > 1) lcls += (float)(v[1] / ((double)n * L.nc));
    }
    lobj += (float)(v[2] / ((double)L.B * L.na * L.ny[l] * L.nx[l])) * L.balance[l];
  }
  if (threadIdx.x == 0) {
    lbox *= L.hyp_box;
    lobj *= L.hyp_obj;
    lcls *= L.hyp_cls;
    out[0] = ((lbox + lobj) + lcls) * (float)L.B;
    out[1] = lbox;
    out[2] = lobj;
    out[3] = lcls;
  }
}

// --------------------------------------------------------------------------------------------------------------------------- backward
// d(loss)/d(obj logit) = g * B * hyp_obj * balance / (B na ny nx) * (sigmoid(x) - tobj): written here with tobj = 0, every other channel 0;
// the candidate cells are rewritten by v5_cell_grad_kernel.
__global__ void __launch_bounds__(kV5Threads) v5_fill_kernel(V5Levels L, int l, const float* __restrict__ gout) {
  const long long hw = (long long)L.ny[l] * L.nx[l], no = 5 + L.nc, n = (long long)L.B * L.na * no * hw;
  const float s_obj = gout[0] * (float)L.B * L.hyp_obj * L.balance[l] / (float)((double)L.B * L.na * hw);
  const float* p = L.p[l];
  float* g = L.g[l];
  for (long long i = blockIdx.x * (long long)kV5Threads + threadIdx.x; i < n; i += (long long)gridDim.x * kV5Threads)
    g[i] = ((i / hw) % no == 4) ? s_obj * sigmoidf(p[i]) : 0.0f;
}

__global__ void __launch_bounds__(kV5Threads) v5_cell_grad_kernel(V5Levels L, const int* __restrict__ cand_idx, const float* __restrict__ cand_box,
                                                                  const int* __restrict__ ncand, const int* __restrict__ key, const int* __restrict__ sorted,
                                                                  const float* __restrict__ score, const float* __restrict__ gout) {
  const int l = blockIdx.y, p = blockIdx.x * kV5Threads + threadIdx.x, n = ncand[l];
  if (p >= n) return;
  const size_t off = (size_t)l * L.cap;
  if (!run_head(sorted + off, key + off, p)) return;
  int q;
  const float t = cell_tobj(L, score + off, sorted + off, key + off, n, p, &q);
  const int* c0 = cand_idx + (off + sorted[off + p]) * 5;
  const size_t hw = (size_t)L.ny[l] * L.nx[l], cb = cell_base(L, l, c0[0], c0[1], c0[2], c0[3]);
  const float* x = L.p[l] + cb;
  float* g = L.g[l] + cb;
  const float B = (float)L.B, go = gout[0];
  const float s_box = go * B * L.hyp_box / (float)n;                                   // d(loss) / d(1 - ciou_k)
  const float s_obj = go * B * L.hyp_obj * L.balance[l] / (float)((double)L.B * L.na * hw);
  const float s_cls = go * B * L.hyp_cls / (float)((double)n * L.nc);
  g[4 * hw] = s_obj * (sigmoidf(x[4 * hw]) - t);
  float acc[4] = {0.0f, 0.0f, 0.0f, 0.0f};
  for (int r = p; r <= q; ++r) {  // the cell's candidates in candidate order
    const float* tb = cand_box + (off + sorted[off + r]) * 6;
    const Pred pr = decode(x, hw, tb);
    float d[4];
    ciou(pr.px, pr.py, pr.pw, pr.ph, tb, d);
    const float gc = -s_box;
    // pxy = 2 s - 0.5: 2 s (1 - s); pwh = (2 s)^2 a: 2 (2 s) 2 a s (1 - s)
    acc[0] += gc * d[0] * 2.0f * (pr.sx * (1.0f - pr.sx));
    acc[1] += gc * d[1] * 2.0f * (pr.sy * (1.0f - pr.sy));
    acc[2] += gc * d[2] * tb[4] * 2.0f * (pr.sw * 2.0f) * 2.0f * (pr.sw * (1.0f - pr.sw));
    acc[3] += gc * d[3] * tb[5] * 2.0f * (pr.sh * 2.0f) * 2.0f * (pr.sh * (1.0f - pr.sh));
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) g[i * hw] = acc[i];
  if (L.nc > 1) {
    for (int j = 0; j < L.nc; ++j) {
      const float sj = sigmoidf(x[(5 + j) * hw]);
      float a = 0.0f;
      for (int r = p; r <= q; ++r) a += s_cls * (sj - (cand_idx[(off + sorted[off + r]) * 5 + 4] == j ? 1.0f : 0.0f));
      g[(5 + j) * hw] = a;
    }
  }
}

// --------------------------------------------------------------------------------------------------------------------------- host
struct V5Ws {
  int *key, *sorted;
  float* score;
  double *term, *corr, *partial;
  size_t bytes;
};

V5Ws v5_ws(void* base, int nlev, int cap) {
  WsCarver c(base);
  V5Ws w{};
  const size_t n = (size_t)nlev * (cap > 0 ? cap : 1);
  w.key = static_cast<int*>(c.take(n * 4));
  w.sorted = static_cast<int*>(c.take(n * 4));
  w.score = static_cast<float*>(c.take(n * 4));
  w.term = static_cast<double*>(c.take(n * 2 * sizeof(double)));
  w.corr = static_cast<double*>(c.take(n * sizeof(double)));
  w.partial = static_cast<double*>(c.take((size_t)nlev * kV5ObjBlocks * sizeof(double)));
  w.bytes = c.bytes();
  return w;
}

int make_levels(const char* what, const float* const* preds, const int32_t* shapes, const float* anchors, const float* balance, int32_t nlev, int32_t na,
                int32_t nc, const float* targets, int32_t nt, const float* hyp, float* const* grads, V5Levels* L) {
  CVB_REQUIRE(preds && shapes && anchors && balance && hyp, "%s: preds, shapes, anchors, balance and hyp are required", what);
  CVB_REQUIRE(nlev >= 1 && nlev <= kV5MaxLevels, "%s: 1 to %d levels supported (got %d)", what, kV5MaxLevels, nlev);
  CVB_REQUIRE(na >= 1 && na <= kV5MaxAnchors, "%s: 1 to %d anchors per level supported (got %d)", what, kV5MaxAnchors, na);
  CVB_REQUIRE(nc >= 1, "%s: num_classes must be >= 1 (got %d)", what, nc);
  CVB_REQUIRE(nt >= 0, "%s: nt must be >= 0 (got %d)", what, nt);
  CVB_REQUIRE(nt == 0 || (targets && is_aligned(targets, 4)), "%s: targets [nt, 6] required, 4-byte aligned", what);
  CVB_REQUIRE((long long)5 * na * nt < (1LL << 28), "%s: too many targets (%d)", what, nt);
  CVB_REQUIRE(hyp[0] > 1.0f, "%s: anchor_t must be > 1 (got %g)", what, (double)hyp[0]);
  *L = V5Levels{};
  const int B = shapes[0];
  CVB_REQUIRE(B >= 1, "%s: batch must be >= 1 (got %d)", what, B);
  for (int l = 0; l < nlev; ++l) {
    const int32_t* s = shapes + 4 * l;
    CVB_REQUIRE(preds[l] && is_aligned(preds[l], 4), "%s: level %d output missing or not 4-byte aligned", what, l);
    CVB_REQUIRE(s[0] == B && s[1] == na * (5 + nc) && s[2] > 0 && s[3] > 0,
                "%s: level %d output must be [B=%d, na * (5 + nc)=%d, ny > 0, nx > 0] (got [%d, %d, %d, %d])", what, l, B, na * (5 + nc), s[0], s[1], s[2], s[3]);
    CVB_REQUIRE((long long)B * na * (5 + nc) * s[2] * s[3] < INT_MAX, "%s: level %d too large", what, l);
    if (grads) CVB_REQUIRE(grads[l] && is_aligned(grads[l], 4), "%s: level %d gradient missing or not 4-byte aligned", what, l);
    for (int a = 0; a < na; ++a) {
      const float aw = anchors[(l * na + a) * 2], ah = anchors[(l * na + a) * 2 + 1];
      CVB_REQUIRE(aw > 0.0f && ah > 0.0f, "%s: level %d anchor %d must be positive (got %g x %g)", what, l, a, (double)aw, (double)ah);
      L->anchor[l][a][0] = aw;
      L->anchor[l][a][1] = ah;
    }
    L->p[l] = preds[l];
    L->g[l] = grads ? grads[l] : nullptr;
    L->ny[l] = s[2];
    L->nx[l] = s[3];
    L->balance[l] = balance[l];
  }
  L->nlev = nlev;
  L->na = na;
  L->nc = nc;
  L->B = B;
  L->nt = nt;
  L->cap = 5 * na * nt;
  L->anchor_t = hyp[0];
  L->hyp_box = hyp[1];
  L->hyp_obj = hyp[2];
  L->hyp_cls = hyp[3];
  L->gr = hyp[4];
  return CVB_OK;
}

int check_outputs(const char* what, const int32_t* cand_idx, const float* cand_box, const int32_t* ncand, const void* workspace, size_t ws_bytes, const V5Levels& L) {
  CVB_REQUIRE(cand_idx && cand_box && ncand && is_aligned(cand_idx, 4) && is_aligned(cand_box, 4) && is_aligned(ncand, 4),
              "%s: cand_idx, cand_box and ncand are required, 4-byte aligned", what);
  const size_t need = v5_ws(nullptr, L.nlev, L.cap).bytes;
  CVB_REQUIRE(workspace && is_aligned(workspace, 256), "%s: workspace required, 256-byte aligned", what);
  CVB_REQUIRE(ws_bytes >= need, "%s: workspace of %zu bytes too small (%zu needed)", what, ws_bytes, need);
  return CVB_OK;
}

}  // namespace
}  // namespace cvb

using namespace cvb;

extern "C" size_t cvb_train_yolov5_loss_workspace_bytes(int32_t nlev, int32_t na, int32_t nt) {
  if (nlev < 1 || nlev > kV5MaxLevels || na < 1 || na > kV5MaxAnchors || nt < 0) return 0;
  return v5_ws(nullptr, nlev, 5 * na * nt).bytes;
}

extern "C" int cvb_train_yolov5_loss_fwd(const float* const* preds, const int32_t* shapes, const float* anchors, const float* balance, int32_t nlev, int32_t na,
                                         int32_t nc, const float* targets, int32_t nt, const float* hyp, int32_t* cand_idx, float* cand_box, int32_t* ncand,
                                         float* out, void* workspace, size_t ws_bytes, void* stream) {
  V5Levels L;
  int rc = make_levels("train_yolov5_loss_fwd", preds, shapes, anchors, balance, nlev, na, nc, targets, nt, hyp, nullptr, &L);
  if (rc != CVB_OK) return rc;
  rc = check_outputs("train_yolov5_loss_fwd", cand_idx, cand_box, ncand, workspace, ws_bytes, L);
  if (rc != CVB_OK) return rc;
  CVB_REQUIRE(out && is_aligned(out, 4), "train_yolov5_loss_fwd: out [4] required, 4-byte aligned");
  const V5Ws w = v5_ws(workspace, nlev, L.cap);
  cudaStream_t st = as_stream(stream);
  const int cblk = ceil_div(L.cap > 0 ? L.cap : 1, kV5Threads);
  v5_cand_kernel<<<nlev, 1024, 0, st>>>(L, targets, cand_idx, cand_box, ncand, w.key);
  v5_rank_kernel<<<dim3(cblk, nlev), kV5Threads, 0, st>>>(L.cap, w.key, ncand, w.sorted);
  v5_term_kernel<<<dim3(cblk, nlev), kV5Threads, 0, st>>>(L, cand_idx, cand_box, ncand, w.score, w.term);
  v5_seg_kernel<<<dim3(cblk, nlev), kV5Threads, 0, st>>>(L, cand_idx, ncand, w.key, w.sorted, w.score, w.corr);
  v5_obj_kernel<<<dim3(kV5ObjBlocks, nlev), kV5Threads, 0, st>>>(L, w.partial);
  v5_final_kernel<<<1, kV5Threads, 0, st>>>(L, ncand, w.term, w.corr, w.partial, out);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch(6);
  return CVB_OK;
}

extern "C" int cvb_train_yolov5_loss_bwd(const float* const* preds, const int32_t* shapes, const float* anchors, const float* balance, int32_t nlev, int32_t na,
                                         int32_t nc, const float* targets, int32_t nt, const float* hyp, const int32_t* cand_idx, const float* cand_box,
                                         const int32_t* ncand, const void* workspace, size_t ws_bytes, const float* grad_out, float* const* grads, void* stream) {
  CVB_REQUIRE(grads, "train_yolov5_loss_bwd: grads required");
  V5Levels L;
  int rc = make_levels("train_yolov5_loss_bwd", preds, shapes, anchors, balance, nlev, na, nc, targets, nt, hyp, grads, &L);
  if (rc != CVB_OK) return rc;
  rc = check_outputs("train_yolov5_loss_bwd", cand_idx, cand_box, ncand, workspace, ws_bytes, L);
  if (rc != CVB_OK) return rc;
  CVB_REQUIRE(grad_out && is_aligned(grad_out, 4), "train_yolov5_loss_bwd: grad_out [1] required, 4-byte aligned");
  const V5Ws w = v5_ws(const_cast<void*>(workspace), nlev, L.cap);
  cudaStream_t st = as_stream(stream);
  for (int l = 0; l < nlev; ++l) {
    const long long n = (long long)L.B * na * (5 + nc) * L.ny[l] * L.nx[l];
    v5_fill_kernel<<<(int)std::min<long long>((n + kV5Threads - 1) / kV5Threads, 8LL * kSmCount), kV5Threads, 0, st>>>(L, l, grad_out);
  }
  const int cblk = ceil_div(L.cap > 0 ? L.cap : 1, kV5Threads);
  v5_cell_grad_kernel<<<dim3(cblk, nlev), kV5Threads, 0, st>>>(L, cand_idx, cand_box, ncand, w.key, w.sorted, w.score, grad_out);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch(nlev + 1);
  return CVB_OK;
}
