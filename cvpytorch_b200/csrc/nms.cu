// Batched YOLOv5 non-max suppression, all images in flight at once, no host synchronisation.
//
// Replaces the reference's Python loop over images (src/models/yolov5.py:87-151: ~15 ATen launches + one
// torchvision.ops.nms with a device->host sync per image).  Semantics reproduced bit-for-bit:
//   * candidate = anchor with obj > conf (yolov5.py:71,90); conf = cls*obj in fp32 (:106); multi_label keeps every
//     (anchor, class) with conf > thres in nonzero() row-major order (:112-114), else best class (:116-117)
//   * if more than max_nms candidates: keep the max_nms highest scores (:131-132)
//   * boxes: xywh2xyxy in fp32 (:52-59), class offset cls*max_wh added in fp32 (:135-136)
//   * torchvision.ops.nms (third-party, v0.7..0.26 identical): stable sort by score descending (ties: lower
//     candidate index first), greedy, suppress when  inter/(a_i+a_j-inter) > iou_thres  with the comparison done
//     in DOUBLE (the CPU kernel compares the float IoU against the double threshold), areas without +1
//   * at most max_det rows returned (:138-139).  Greedy NMS only needs candidates in score order until max_det
//     boxes are kept, so the scan stops early; the output is identical to truncating the full keep list.
//
// Pipeline: histogram of score bits -> per-image threshold bin (top max_nms) -> emit 64-bit keys
// (score bits << 32 | ~candidate id) -> segmented bitonic sort (descending; shared-memory fused below 4096)
// -> per-image greedy scan (warp-ballot compaction, 512x512 bit mask in shared memory, single-warp resolve).
#include <cooperative_groups.h>
#include <cuda_fp16.h>
#include <math_constants.h>

#include "internal.h"

namespace cvb {

constexpr int kBins = kNmsBins;  // nms_score_bin (internal.h)
constexpr int kCap = kNmsCap;  // candidate key capacity per image
constexpr int kChunk = 4096;   // keys sorted per CTA in shared memory
constexpr int kGreedyThreads = 512;

constexpr int kCapA = kNmsCapA;  // phase-A (early exit) candidate capacity = one shared-memory sort chunk
constexpr int kTargetA = 3072; // phase A takes the smallest set of top score bins holding >= this many candidates

// Two-phase scheme: greedy NMS only needs candidates in score order until max_det boxes are kept, so phase A runs the
// whole pipeline on the top ~3k candidates (one smem sort chunk per image); only images that did not reach max_det there
// (and have more candidates) go through phase B = the full top-max_nms path.  `done[b]` is decided on the device.
struct NmsWs {
  uint32_t* hist;   // [B][kBins]                          (shared by both phases)
  uint32_t* cnt;    // [B]      candidates emitted in this phase
  uint32_t* tbin;   // [B]      threshold bin of this phase
  uint64_t* keys;   // [B][cap]
  uint32_t* done;   // [B]      set by phase A's greedy kernel
  uint32_t* total;  // [B]      number of candidates of the image (all bins)
  float* rowmax;    // [B][A]   best candidate score of each anchor row (0: none), see internal.h
  int cap;          // kCapA or kCap
  int phase;        // 0 = A, 1 = B
};

static NmsWs carve_ws(void* ws, int B, int phase) {
  NmsWs w;
  uint8_t* p = static_cast<uint8_t*>(ws);
  const size_t slot = align_up((size_t)B * 4, 256);
  w.hist = reinterpret_cast<uint32_t*>(p);
  p += align_up((size_t)B * kBins * 4, 256);
  uint32_t* cntB = reinterpret_cast<uint32_t*>(p);
  uint32_t* tbinB = reinterpret_cast<uint32_t*>(p + slot);
  uint32_t* cntA = reinterpret_cast<uint32_t*>(p + 2 * slot);
  uint32_t* tbinA = reinterpret_cast<uint32_t*>(p + 3 * slot);
  w.done = reinterpret_cast<uint32_t*>(p + 4 * slot);
  w.total = reinterpret_cast<uint32_t*>(p + 5 * slot);
  p += 6 * slot;
  uint64_t* keysB = reinterpret_cast<uint64_t*>(p);
  uint64_t* keysA = keysB + (size_t)B * kCap;
  w.rowmax = nms_ws_rowmax(ws, B);
  w.phase = phase;
  if (phase == 0) {
    w.cnt = cntA;
    w.tbin = tbinA;
    w.keys = keysA;
    w.cap = kCapA;
  } else {
    w.cnt = cntB;
    w.tbin = tbinB;
    w.keys = keysB;
    w.cap = kCap;
  }
  return w;
}

// ------------------------------------------------------------------ building blocks of the YOLOv5, YOLOX and FCOS pipelines
// Sort key of a candidate: score bits above, ~id below.  Scores are non-negative, so descending key order is descending score
// with ties broken by the lower id (torchvision's stable order), and no two keys are equal.
__device__ __forceinline__ uint64_t make_key(uint32_t score_bits, uint32_t id) {
  return ((uint64_t)score_bits << 32) | (uint64_t)(0xFFFFFFFFu - id);
}
__device__ __forceinline__ uint32_t key_id(uint64_t key) { return 0xFFFFFFFFu - (uint32_t)(key & 0xFFFFFFFFull); }
__device__ __forceinline__ float key_score(uint64_t key) { return __uint_as_float((uint32_t)(key >> 32)); }

// Largest score(c), c in [0, nc), over the warp, returned in `best`, and its class: the first maximum wins, like torch.max.
template <class Score>
__device__ __forceinline__ int warp_argmax_first(int nc, Score score, float& best) {
  const int lane = threadIdx.x & 31;
  best = -1.0f;
  int bi = 0x7fffffff;
  for (int c = lane; c < nc; c += 32) {
    const float s = score(c);
    if (s > best) {
      best = s;
      bi = c;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ob > best || (ob == best && oi < bi)) {
      best = ob;
      bi = oi;
    }
  }
  return bi;
}

// Warp-aggregated append: the lanes with `pass` take consecutive slots, in lane order, from one atomicAdd on *counter.
// Returns the lane's slot (meaningless where !pass).  The whole warp calls it.
__device__ __forceinline__ uint32_t warp_append(uint32_t* counter, bool pass) {
  const int lane = threadIdx.x & 31;
  const uint32_t m = __ballot_sync(0xffffffffu, pass);
  if (m == 0) return 0;
  uint32_t base = 0;
  if (lane == 0) base = atomicAdd(counter, (uint32_t)__popc(m));
  base = __shfl_sync(0xffffffffu, base, 0);
  return base + __popc(m & ((1u << lane) - 1));
}

// Max of v over the block, returned to every thread.  The whole block calls it; red holds one float per warp.
template <int kThreads>
__device__ __forceinline__ float block_max(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float m = red[0];
  for (int w = 1; w < kThreads / 32; ++w) m = fmaxf(m, red[w]);
  return m;
}

// Top-k threshold of a score histogram (global or shared): the highest bin t whose bins [t, kBins) hold >= target candidates,
// 0 when the whole histogram holds fewer.  Warp 0 writes it to *tbin and the histogram's total to *total (when given).  The
// whole block of kThreads calls it; seg is kBins / 32 words of shared memory.
template <int kThreads>
__device__ __forceinline__ void top_bin_search(const uint32_t* hist, uint32_t target, uint32_t* seg, uint32_t* tbin, uint32_t* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int sgi = warp; sgi < kBins / 32; sgi += kThreads / 32) {  // sums of 32-bin segments (coalesced reads, one warp reduction each)
    uint32_t v = hist[sgi * 32 + lane];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) seg[sgi] = v;
  }
  __syncthreads();
  if (warp != 0) return;
  // top-down scan: lane l owns the kPer consecutive segments just below those of lane l-1
  constexpr int kPer = kBins / 32 / 32;
  const int top = kBins / 32 - 1 - lane * kPer;
  uint32_t part = 0;
  for (int i = 0; i < kPer; ++i) part += seg[top - i];
  uint32_t incl = part;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t u = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += u;
  }
  const uint32_t sum = __shfl_sync(0xffffffffu, incl, 31);
  if (lane == 0) {
    *tbin = 0;  // default: everything
    if (total) *total = sum;
  }
  __syncwarp();
  uint32_t run = incl - part;  // candidates in all higher segments
  if (run < target && incl >= target) {  // exactly one lane crosses the target
    for (int i = 0; i < kPer; ++i) {
      const int sgi = top - i;
      if (run + seg[sgi] >= target) {
        for (int j = 31; j >= 0; --j) {
          run += hist[sgi * 32 + j];
          if (run >= target) {
            *tbin = (uint32_t)(sgi * 32 + j);
            break;
          }
        }
        break;
      }
      run += seg[sgi];
    }
  }
}

__device__ __forceinline__ void cmpswap(uint64_t* s, int i, int l, bool desc) {
  const uint64_t x = s[i], y = s[l];
  if (desc ? (x < y) : (x > y)) {
    s[i] = y;
    s[l] = x;
  }
}

// Stages k = k_lo .. k_hi (powers of two) of a bitonic sort, run on the n keys s = keys[start, start + n) of the sequence held in
// shared memory (n a power of two), steps j < n only: steps j >= n pair keys of different tiles and run elsewhere.  The pair
// (i, i + j) is put in descending order where ((start + i) & k) == 0, ascending elsewhere.  The caller syncs before it reads s.
__device__ __forceinline__ void bitonic_tile(uint64_t* s, int n, uint32_t start, int k_lo, int k_hi) {
  for (int k = k_lo; k <= k_hi; k <<= 1)
    for (int j = min(k, n) >> 1; j > 0; j >>= 1) {
      __syncthreads();
      for (int t = threadIdx.x; t < n / 2; t += blockDim.x) {
        const int i = 2 * j * (t / j) + (t % j);
        cmpswap(s, i, i + j, ((start + i) & k) == 0);
      }
    }
}

// Torchvision's IoU test: fp32 IoU, areas without +1, compared in double against the threshold
__device__ __forceinline__ bool iou_gt(const float4& a, float aa, const float4& b, float ab, double thr) {
  const float xx1 = fmaxf(a.x, b.x), yy1 = fmaxf(a.y, b.y);
  const float xx2 = fminf(a.z, b.z), yy2 = fminf(a.w, b.w);
  const float w = fmaxf(0.0f, __fsub_rn(xx2, xx1));
  const float h = fmaxf(0.0f, __fsub_rn(yy2, yy1));
  const float inter = __fmul_rn(w, h);
  const float ovr = __fdiv_rn(inter, __fsub_rn(__fadd_rn(aa, ab), inter));
  return (double)ovr > thr;
}

// Greedy NMS over candidates in score order, one chunk of kChunk at a time.
template <int kChunk>
struct GreedyChunk {
  float4 box[kChunk];  // the chunk's survivors, compacted in score order: boxes as the suppression rule sees them
  float area[kChunk];
  int cls[kChunk];
  uint32_t payload[kChunk];            // the caller's handle of the candidate
  uint32_t mask[kChunk][kChunk / 32];  // bit c of row r: survivor r suppresses survivor c > r
  uint32_t keep[kChunk];               // rows kept by the resolve, in order
  uint32_t warp_cnt[32];
  uint32_t m, nk;
};

// Thread t < kChunk holds the chunk's candidate t; it is not `alive` past the end of the list or when a box kept in an earlier
// chunk suppresses it.  The survivors are compacted in order, suppress(r, c) (survivor r < c of G suppresses c) fills the bit mask,
// and one warp resolves it in order, keeping at most `limit` rows.  Returns the number kept; G.keep lists their rows.  The caller syncs before G is reused.
template <int kThreads, int kChunk, class Suppress>
__device__ __forceinline__ int greedy_chunk(GreedyChunk<kChunk>& G, bool alive, const float4& box, float area, int cls, uint32_t payload,
                                            int limit, Suppress suppress) {
  static_assert(kThreads >= kChunk && kThreads <= 1024, "one thread per candidate of the chunk");
  constexpr int kWarps = kThreads / 32;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // order-preserving compaction of the survivors
  const uint32_t bal = __ballot_sync(0xffffffffu, alive);
  if (lane == 0) G.warp_cnt[warp] = __popc(bal);
  __syncthreads();
  if (warp == 0) {
    const uint32_t v = (lane < kWarps) ? G.warp_cnt[lane] : 0;
    uint32_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t u = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += u;
    }
    if (lane < kWarps) G.warp_cnt[lane] = inc - v;
    if (lane == 31) G.m = inc;
  }
  __syncthreads();
  const int m = (int)G.m;
  if (alive) {
    const int pos = (int)G.warp_cnt[warp] + __popc(bal & ((1u << lane) - 1));
    G.box[pos] = box;
    G.area[pos] = area;
    G.cls[pos] = cls;
    G.payload[pos] = payload;
  }
  __syncthreads();
  // suppression bit mask among the m survivors (row r suppresses column c > r)
  const int words = (m + 31) >> 5;
  if (tid < m) {
    for (int wd = 0; wd < words; ++wd) {
      uint32_t bits = 0;
      const int c0 = wd << 5, c1 = min(m, c0 + 32);
      for (int c = max(c0, tid + 1); c < c1; ++c)
        if (suppress(tid, c)) bits |= 1u << (c & 31);
      G.mask[tid][wd] = bits;
    }
  }
  __syncthreads();
  // sequential greedy resolve by one warp; lane l owns word l of the "removed" bitset
  if (warp == 0) {
    uint32_t removed = 0;
    int nk = 0;
    for (int r = 0; r < m && nk < limit; ++r) {
      const uint32_t rw = __shfl_sync(0xffffffffu, removed, r >> 5);
      if (!((rw >> (r & 31)) & 1u)) {
        if (lane == 0) G.keep[nk] = (uint32_t)r;
        ++nk;
        if (lane < words) removed |= G.mask[r][lane];
      }
    }
    if (lane == 0) G.nk = (uint32_t)nk;
  }
  __syncthreads();
  return (int)G.nk;
}

// ------------------------------------------------------------------ counting pass (only when the decode kernel did not build the histogram)
// Grid (ceil(A / kRowsPerCta), B); each warp walks rows of ONE image: histogram of score bits (spread global atomics) and the
// per-row best score (rowmax) that lets the emit passes skip rows.  MULTI: multi-label histogram.  At most 32 registers (8 CTAs per SM):
// uncapped, the multi-label kernel takes 44.
constexpr int kRowsPerCta = 64;
constexpr int kScanThreads = 256;

template <bool MULTI>
__global__ void __launch_bounds__(kScanThreads, 8) nms_count_kernel(const float* __restrict__ pred, int A, int nc, float conf, NmsWs ws) {
  const int no = nc + 5;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int b = blockIdx.y;
  const int row0 = blockIdx.x * kRowsPerCta;
  const int row1 = min(A, row0 + kRowsPerCta);
  float* rowmax = ws.rowmax + (size_t)b * A;
  uint32_t* hist = ws.hist + (size_t)b * kBins;
  constexpr int R = 4;  // rows in flight per warp: all loads of a batch are issued before the first use
  for (int base = row0 + warp * R; base < row1; base += (kScanThreads / 32) * R) {
    float obj[R];
#pragma unroll
    for (int i = 0; i < R; ++i) {
      const int anchor = min(base + i, row1 - 1);
      obj[i] = __ldg(pred + ((size_t)b * A + anchor) * no + 4);
    }
    for (int i = 0; i < R; ++i) {
      const int anchor = base + i;
      if (anchor >= row1) continue;
      if (!(obj[i] > conf)) {
        if (lane == 0) rowmax[anchor] = 0.0f;
        continue;
      }
      const float* r = pred + ((size_t)b * A + anchor) * no;
      float rbest = 0.0f;
      for (int c = lane; c < nc; c += 32) nms_count_score(hist, yolo_score(__ldg(r + 5 + c), obj[i]), conf, MULTI, rbest);
      rbest = nms_finish_row(hist, rbest, conf, MULTI, lane);
      if (lane == 0) rowmax[anchor] = rbest;
    }
  }
}

// ------------------------------------------------------------------ emit pass (both phases)
// Grid (ceil(A / kEmitRows), B).  Step 1: one coalesced read of the CTA's rowmax slice builds the list of live rows (best score
// in or above the threshold bin) in shared memory -- in phase A that is a few percent of the rows, so almost nothing of the
// 548 MB prediction tensor is touched.  Step 2: the warps walk the live rows in batches of kRowsPerCta (the staging buffer's
// worst case), recompute obj*cls exactly as the counting pass did, stage the keys and copy each batch out with one global
// atomic.  Key order inside the image's array is irrelevant (unique keys, sorted next).
constexpr int kEmitRows = 512;

__global__ void __launch_bounds__(kScanThreads) nms_emit_kernel(const float* __restrict__ pred, int A, int nc, float conf, int multi_label,
                                                                NmsWs ws, int* __restrict__ status) {
  extern __shared__ uint64_t stage[];  // [kRowsPerCta * nc] worst case of one batch
  __shared__ uint32_t s_cnt, s_base, s_nlive;
  __shared__ int s_live[kEmitRows];
  const int no = nc + 5;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int b = blockIdx.y;
  if (ws.phase == 1 && ws.done[b]) return;  // phase A already produced this image's result
  const uint32_t tb = ws.tbin[b];
  const float* rowmax = ws.rowmax + (size_t)b * A;
  const int row0 = blockIdx.x * kEmitRows;
  if (threadIdx.x == 0) s_nlive = 0;
  __syncthreads();
  for (int r = threadIdx.x; r < kEmitRows; r += kScanThreads) {
    const int row = row0 + r;
    if (row < A) {
      const float rm = __ldg(rowmax + row);
      if (__float_as_uint(rm) != 0u && nms_score_bin(rm) >= tb) s_live[atomicAdd(&s_nlive, 1u)] = row;
    }
  }
  __syncthreads();
  const int nlive = (int)s_nlive;
  for (int batch0 = 0; batch0 < nlive; batch0 += kRowsPerCta) {  // uniform trip count
    if (threadIdx.x == 0) s_cnt = 0;
    __syncthreads();
    const int batch1 = min(nlive, batch0 + kRowsPerCta);
    if (multi_label && nc <= 96) {
      // hot configuration: R live rows per warp in flight, objectness and the three class chunks of every row requested
      // together (a live row always passes obj > conf), so a CTA pays about one DRAM latency per batch
      constexpr int R = 4, NW = kScanThreads / 32;
      for (int l0 = batch0 + warp; l0 < batch1; l0 += NW * R) {
        float v[R][3], ob[R];
        int an[R];
#pragma unroll
        for (int i = 0; i < R; ++i) {
          const int li = l0 + i * NW;
          an[i] = s_live[min(li, batch1 - 1)];
          const float* r = pred + ((size_t)b * A + an[i]) * no;
          ob[i] = __ldg(r + 4);
#pragma unroll
          for (int k = 0; k < 3; ++k) {
            const int c = k * 32 + lane;
            v[i][k] = (c < nc) ? __ldg(r + 5 + c) : 0.0f;
          }
        }
#pragma unroll
        for (int i = 0; i < R; ++i) {
          if (l0 + i * NW >= batch1 || !(ob[i] > conf)) continue;  // warp-uniform
#pragma unroll
          for (int k = 0; k < 3; ++k) {
            const int c = k * 32 + lane;
            const float sc = (c < nc) ? yolo_score(v[i][k], ob[i]) : 0.0f;
            const bool pass = c < nc && sc > conf && nms_score_bin(sc) >= tb;
            const uint32_t slot = warp_append(&s_cnt, pass);
            if (pass) stage[slot] = make_key(__float_as_uint(sc), (uint32_t)an[i] * (uint32_t)nc + (uint32_t)c);
          }
        }
      }
    } else
    for (int li = batch0 + warp; li < batch1; li += kScanThreads / 32) {
      const int anchor = s_live[li];
      const float* r = pred + ((size_t)b * A + anchor) * no;
      const float ob = __ldg(r + 4);
      if (!(ob > conf)) continue;  // cannot happen for a live row; kept for symmetry with the counting pass
      if (multi_label) {
        for (int c0 = 0; c0 < nc; c0 += 32) {
          const int c = c0 + lane;
          const float sc = (c < nc) ? yolo_score(__ldg(r + 5 + c), ob) : 0.0f;
          const bool pass = c < nc && sc > conf && nms_score_bin(sc) >= tb;
          const uint32_t slot = warp_append(&s_cnt, pass);
          if (pass) stage[slot] = make_key(__float_as_uint(sc), (uint32_t)anchor * (uint32_t)nc + (uint32_t)c);
        }
      } else {
        // best class only: conf, j = x[:, 5:].max(1)
        float best;
        const int bi = warp_argmax_first(nc, [&](int c) { return yolo_score(__ldg(r + 5 + c), ob); }, best);
        if (lane == 0 && best > conf && nms_score_bin(best) >= tb)
          stage[atomicAdd(&s_cnt, 1u)] = make_key(__float_as_uint(best), (uint32_t)anchor * (uint32_t)nc + (uint32_t)bi);
      }
    }
    __syncthreads();
    const uint32_t n = s_cnt;
    if (n != 0) {  // uniform
      if (threadIdx.x == 0) s_base = atomicAdd(&ws.cnt[b], n);
      __syncthreads();
      const uint32_t base = s_base;
      if (base + n > (uint32_t)ws.cap && ws.phase == 1 && status && threadIdx.x == 0) atomicExch(&status[0], 1);
      uint64_t* keys = ws.keys + (size_t)b * ws.cap;
      for (uint32_t i = threadIdx.x; i < n; i += kScanThreads)
        if (base + i < (uint32_t)ws.cap) keys[base + i] = stage[i];
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------ threshold bin: smallest set of top bins holding >= max_nms
__global__ void __launch_bounds__(256) nms_threshold_kernel(NmsWs ws, int target) {
  __shared__ uint32_t seg[kBins / 32];
  const int b = blockIdx.x;
  top_bin_search<256>(ws.hist + (size_t)b * kBins, (uint32_t)target, seg, &ws.tbin[b], &ws.total[b]);
}

// ------------------------------------------------------------------ segmented bitonic sort (descending)
__device__ __forceinline__ uint32_t seg_npad(const NmsWs& ws, int b, uint32_t* n_out) {
  uint32_t n = ws.cnt[b];
  if (n > (uint32_t)ws.cap) n = ws.cap;
  if (ws.phase == 1 && ws.done[b]) n = 0;  // nothing to sort: every chunk beyond the first returns immediately
  *n_out = n;
  return n <= 1 ? 1u : (1u << (32 - __clz(n - 1)));
}

// full sort of each 4096-key chunk (stages k = 2..4096)
__global__ void __launch_bounds__(1024) bitonic_local_sort_kernel(NmsWs ws) {
  __shared__ uint64_t s[kChunk];
  const int b = blockIdx.y;
  uint32_t n;
  const uint32_t npad = seg_npad(ws, b, &n);
  const uint32_t start = blockIdx.x * kChunk;
  if (start >= npad) return;
  if (ws.phase == 1 && ws.done[b]) return;
  uint64_t* keys = ws.keys + (size_t)b * ws.cap;
  for (int i = threadIdx.x; i < kChunk; i += blockDim.x) s[i] = (start + i < n) ? keys[start + i] : 0ull;
  bitonic_tile(s, kChunk, start, 2, kChunk);
  __syncthreads();
  for (int i = threadIdx.x; i < kChunk; i += blockDim.x) keys[start + i] = s[i];
}

// Phase B in ONE cooperative launch: the whole segmented bitonic sort (local sort, global steps, local merges) with grid-wide
// barriers between steps.  When no image needs phase B (the common case: phase A already kept max_det boxes everywhere) every
// CTA sees that from the `done` flags and returns before the first barrier, so the idle cost is one small launch instead of
// one launch per step.
__global__ void __launch_bounds__(1024) bitonic_full_sort_kernel(NmsWs ws, int B) {
  namespace cg = cooperative_groups;
  cg::grid_group grid = cg::this_grid();
  __shared__ uint64_t s[kChunk];
  __shared__ int s_any;
  if (threadIdx.x == 0) s_any = 0;
  __syncthreads();
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    uint32_t n;
    seg_npad(ws, b, &n);
    if (n > 1) s_any = 1;
  }
  __syncthreads();
  if (!s_any) return;  // identical decision in every CTA: nobody reaches a grid barrier
  constexpr int kChunks = kCap / kChunk;
  // ---- full sort of every 4096-key chunk
  for (int w = blockIdx.x; w < kChunks * B; w += gridDim.x) {
    const int b = w / kChunks;
    const uint32_t start = (uint32_t)(w % kChunks) * kChunk;
    uint32_t n;
    const uint32_t npad = seg_npad(ws, b, &n);
    if (start >= npad) continue;  // uniform per work item
    uint64_t* keys = ws.keys + (size_t)b * ws.cap;
    __syncthreads();
    for (int i = threadIdx.x; i < kChunk; i += blockDim.x) s[i] = (start + i < n) ? keys[start + i] : 0ull;
    bitonic_tile(s, kChunk, start, 2, kChunk);
    __syncthreads();
    for (int i = threadIdx.x; i < kChunk; i += blockDim.x) keys[start + i] = s[i];
  }
  grid.sync();
  for (uint32_t k = 2 * kChunk; k <= (uint32_t)kCap; k <<= 1) {
    for (uint32_t j = k >> 1; j >= (uint32_t)kChunk; j >>= 1) {
      const uint32_t per = kCap / 2;
      for (uint32_t e = blockIdx.x * blockDim.x + threadIdx.x; e < per * (uint32_t)B; e += gridDim.x * blockDim.x) {
        const int b = (int)(e / per);
        const uint32_t t = e - (uint32_t)b * per;
        uint32_t n;
        const uint32_t npad = seg_npad(ws, b, &n);
        if (k > npad) continue;
        const uint32_t i = 2 * j * (t / j) + (t % j);
        if (i >= npad) continue;
        cmpswap(ws.keys + (size_t)b * ws.cap, (int)i, (int)(i + j), (i & k) == 0);
      }
      grid.sync();
    }
    for (int w = blockIdx.x; w < kChunks * B; w += gridDim.x) {
      const int b = w / kChunks;
      const uint32_t start = (uint32_t)(w % kChunks) * kChunk;
      uint32_t n;
      const uint32_t npad = seg_npad(ws, b, &n);
      if (k > npad || start >= npad) continue;
      uint64_t* keys = ws.keys + (size_t)b * ws.cap;
      __syncthreads();
      for (int i = threadIdx.x; i < kChunk; i += blockDim.x) s[i] = keys[start + i];
      bitonic_tile(s, kChunk, start, (int)k, (int)k);
      __syncthreads();
      for (int i = threadIdx.x; i < kChunk; i += blockDim.x) keys[start + i] = s[i];
    }
    grid.sync();
  }
}

// ------------------------------------------------------------------ greedy scan
using GreedySmem = GreedyChunk<kGreedyThreads>;

// xywh2xyxy of one prediction row in fp32 (yolov5.py:52-59)
__device__ __forceinline__ float4 row_xyxy(const float* r) {
  const float cx = __ldg(r), cy = __ldg(r + 1), w = __ldg(r + 2), h = __ldg(r + 3);
  const float hw = __fmul_rn(w, 0.5f), hh = __fmul_rn(h, 0.5f);
  return make_float4(__fsub_rn(cx, hw), __fsub_rn(cy, hh), __fadd_rn(cx, hw), __fadd_rn(cy, hh));
}

__global__ void __launch_bounds__(kGreedyThreads) nms_greedy_kernel(const float* __restrict__ pred, int A, int nc, NmsWs ws,
                                                                     double iou_thr, int max_nms, int max_det, float max_wh,
                                                                     float* __restrict__ det, int* __restrict__ det_idx,
                                                                     int* __restrict__ det_count) {
  extern __shared__ uint8_t gs_raw[];
  GreedySmem& G = *reinterpret_cast<GreedySmem*>(gs_raw);
  float4* kbox = reinterpret_cast<float4*>(gs_raw + sizeof(GreedySmem));  // [max_det]
  float* karea = reinterpret_cast<float*>(kbox + max_det);                // [max_det]

  const int b = blockIdx.x;
  const int tid = threadIdx.x;
  const int no = nc + 5;
  if (ws.phase == 1 && ws.done[b]) return;
  uint32_t n = ws.cnt[b];
  if (ws.phase == 0 && n > (uint32_t)ws.cap) {  // phase A overflowed its chunk: its key set is incomplete, leave it to phase B
    if (tid == 0) ws.done[b] = 0;
    return;
  }
  if (n > (uint32_t)ws.cap) n = ws.cap;
  if (n > (uint32_t)max_nms) n = max_nms;
  const uint64_t* keys = ws.keys + (size_t)b * ws.cap;
  const float* predb = pred + (size_t)b * A * no;
  int kept_n = 0;

  for (uint32_t base = 0; base < n && kept_n < max_det; base += kGreedyThreads) {
    const uint32_t i = base + tid;
    bool alive = i < n;
    float4 box = make_float4(0, 0, 0, 0);
    float area = 0.0f;
    if (alive) {
      const uint32_t id = key_id(keys[i]);
      const float4 b0 = row_xyxy(predb + (size_t)(id / (uint32_t)nc) * no);
      const float off = __fmul_rn((float)(id % (uint32_t)nc), max_wh);
      box = make_float4(__fadd_rn(b0.x, off), __fadd_rn(b0.y, off), __fadd_rn(b0.z, off), __fadd_rn(b0.w, off));
      area = __fmul_rn(__fsub_rn(box.z, box.x), __fsub_rn(box.w, box.y));
      // suppressed by an already kept (higher score) box?
      for (int k = 0; k < kept_n; ++k) {
        if (iou_gt(kbox[k], karea[k], box, area, iou_thr)) {
          alive = false;
          break;
        }
      }
    }
    const int nk = greedy_chunk<kGreedyThreads>(G, alive, box, area, 0, i, max_det - kept_n,
                                                [&](int r, int c) { return iou_gt(G.box[r], G.area[r], G.box[c], G.area[c], iou_thr); });
    // append to the kept list and write the detections; the payload is the candidate's key position
    for (int t = tid; t < nk; t += kGreedyThreads) {
      const int r = (int)G.keep[t];
      const int o = kept_n + t;
      kbox[o] = G.box[r];
      karea[o] = G.area[r];
      const uint64_t key = keys[G.payload[r]];
      const uint32_t id = key_id(key);
      const float4 b0 = row_xyxy(predb + (size_t)(id / (uint32_t)nc) * no);
      float* d = det + ((size_t)b * max_det + o) * 6;
      d[0] = b0.x;
      d[1] = b0.y;
      d[2] = b0.z;
      d[3] = b0.w;
      d[4] = key_score(key);
      d[5] = (float)(id % (uint32_t)nc);
      det_idx[(size_t)b * max_det + o] = (int)id;
    }
    kept_n += nk;
    __syncthreads();
  }
  if (tid == 0) {
    det_count[b] = kept_n;
    // phase A is final when max_det boxes were kept, or when it already saw every candidate of the image
    if (ws.phase == 0) ws.done[b] = (kept_n >= max_det || ws.cnt[b] == ws.total[b]) ? 1u : 0u;
  }
}

}  // namespace cvb

using namespace cvb;

extern "C" size_t cvb_nms_workspace_bytes(int32_t B, int32_t A, int32_t nc) {
  (void)nc;
  if (B <= 0 || A <= 0) return 0;
  return nms_ws_rowmax_offset(B) + align_up((size_t)B * A * sizeof(float), 256);
}

extern "C" int cvb_nms_workspace_reset(void* workspace, size_t workspace_bytes, int32_t B, void* stream) {
  CVB_REQUIRE(workspace && B > 0 && workspace_bytes >= cvb_nms_workspace_bytes(B, 1, 1), "nms reset: bad workspace");
  CVB_CHECK_CUDA(cudaMemsetAsync(workspace, 0, nms_ws_head_bytes(B), as_stream(stream)));
  return CVB_OK;
}

extern "C" int cvb_yolo_nms(const float* prediction, const CvbNmsParams* p, float* det, int32_t* det_idx, int32_t* det_count,
                            void* workspace, size_t workspace_bytes, int32_t* status, void* stream) {
  CVB_REQUIRE(prediction && p && det && det_idx && det_count && workspace, "nms: null argument");
  CVB_REQUIRE(p->B > 0 && p->A > 0 && p->nc > 0, "nms: bad shape");
  CVB_REQUIRE(p->max_det > 0 && p->max_det <= 4096 && p->max_nms > 0, "nms: bad limits");
  CVB_REQUIRE((long long)p->A * p->nc < 0x7fffffffLL, "nms: candidate id overflow");
  CVB_REQUIRE(workspace_bytes >= cvb_nms_workspace_bytes(p->B, p->A, p->nc), "nms: workspace too small");
  CVB_REQUIRE(is_aligned(workspace, 256), "nms: workspace must be 256-byte aligned");
  cudaStream_t st = as_stream(stream);
  const int multi_label = p->multi_label && p->nc > 1;  // the reference's multi_label &= nc > 1 (include/cvb200.h)
  NmsWs wsA = carve_ws(workspace, p->B, 0), wsB = carve_ws(workspace, p->B, 1);
  if (!p->hist_ready) CVB_CHECK_CUDA(cudaMemsetAsync(workspace, 0, nms_ws_head_bytes(p->B), st));
  if (status) CVB_CHECK_CUDA(cudaMemsetAsync(status, 0, 4 * sizeof(int32_t), st));
  CVB_CHECK_CUDA(cudaMemsetAsync(det, 0, (size_t)p->B * p->max_det * 6 * sizeof(float), st));
  CVB_CHECK_CUDA(cudaMemsetAsync(det_idx, 0xFF, (size_t)p->B * p->max_det * sizeof(int32_t), st));

  dim3 sgrid(ceil_div(p->A, kRowsPerCta), p->B);
  dim3 egrid(ceil_div(p->A, kEmitRows), p->B);
  const size_t stage_bytes = (size_t)kRowsPerCta * p->nc * sizeof(uint64_t);
  CVB_REQUIRE(stage_bytes <= 160 * 1024, "nms: too many classes (%d) for the shared-memory candidate stage", p->nc);
  const size_t gsmem = sizeof(GreedySmem) + (size_t)p->max_det * (sizeof(float4) + sizeof(float));
  CVB_REQUIRE(gsmem <= 200 * 1024, "nms: max_det too large");
  // one-time, thread-safe (C++11 static initialisation) opt-in to the large dynamic shared memory carve-out
  static const cudaError_t emit_smem_err = opt_in_smem(nms_emit_kernel, 160 * 1024);
  static const cudaError_t greedy_smem_err = opt_in_smem(nms_greedy_kernel, 200 * 1024);
  CVB_CHECK_CUDA(emit_smem_err);
  CVB_CHECK_CUDA(greedy_smem_err);
  if (!p->hist_ready) {
    (multi_label ? nms_count_kernel<true> : nms_count_kernel<false>)<<<sgrid, kScanThreads, 0, st>>>(prediction, p->A, p->nc, p->conf_thres, wsB);
    count_launch();
  }
  // ---- phase A: the top ~3k candidates of every image (one shared-memory sort chunk), early exit at max_det
  const int targetA = p->max_nms < kTargetA ? p->max_nms : kTargetA;
  nms_threshold_kernel<<<p->B, 256, 0, st>>>(wsA, targetA);
  nms_emit_kernel<<<egrid, kScanThreads, stage_bytes, st>>>(prediction, p->A, p->nc, p->conf_thres, multi_label, wsA, status);
  bitonic_local_sort_kernel<<<dim3(1, p->B), 1024, 0, st>>>(wsA);
  nms_greedy_kernel<<<p->B, kGreedyThreads, gsmem, st>>>(prediction, p->A, p->nc, wsA, p->iou_thres, p->max_nms, p->max_det, p->max_wh, det,
                                                         det_idx, det_count);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch(4);
  // ---- phase B: full top-max_nms path for the images phase A could not finish (every kernel returns at once otherwise)
  nms_threshold_kernel<<<p->B, 256, 0, st>>>(wsB, p->max_nms);
  nms_emit_kernel<<<egrid, kScanThreads, stage_bytes, st>>>(prediction, p->A, p->nc, p->conf_thres, multi_label, wsB, status);
  count_launch(2);
  {
    // one CTA per SM: co-residency is guaranteed (required by the grid barriers); resolved once, thread-safe static initialisation
    static const int coop_grid = [] {
      const int sms = sm_count();
      int per_sm = 0;
      if (sms == 0 || cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, bitonic_full_sort_kernel, 1024, 0) != cudaSuccess) return 0;
      return per_sm > 0 ? sms : 0;
    }();
    CVB_REQUIRE(coop_grid > 0, "nms: cooperative sort kernel cannot be resident");
    int Bn = p->B;
    void* cargs[2] = {&wsB, &Bn};
    CVB_CHECK_CUDA(cudaLaunchCooperativeKernel(reinterpret_cast<const void*>(bitonic_full_sort_kernel), dim3(coop_grid), dim3(1024), cargs, 0, st));
    count_launch();
  }
  nms_greedy_kernel<<<p->B, kGreedyThreads, gsmem, st>>>(prediction, p->A, p->nc, wsB, p->iou_thres, p->max_nms, p->max_det, p->max_wh, det,
                                                         det_idx, det_count);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}


// =====================================================================================================================
// YOLOX post-processing (src/models/yolox.py:18-68; torchvision.ops.batched_nms at :64 is third-party, un-vendored)
// =====================================================================================================================
namespace cvb {

// One warp per head location.  Record = (x1, y1, x2, y2, obj, class_conf, class_pred, obj * class_conf):
//   xy = (p + grid) * stride, wh = exp(p) * stride (:33-35), sigmoid on obj / classes (:37-39), corners = c -/+ wh / 2 (:46-51),
//   class_conf, class_pred = max over the class sigmoids, first maximum wins (:57).
__global__ void __launch_bounds__(256) yolox_decode_kernel(const float* __restrict__ ro, int ro_pitch, const float* __restrict__ cls, int cls_pitch,
                                                           int B, int H, int W, int nc, float stride, float* __restrict__ cand, long long A,
                                                           long long off) {
  const int lane = threadIdx.x & 31;
  const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const long long npix = (long long)B * H * W;
  if (warp >= npix) return;
  const int hw = H * W;
  const int b = (int)(warp / hw);
  const int p = (int)(warp - (long long)b * hw);
  const int py = p / W, px = p - py * W;
  const float* c = cls + (size_t)warp * cls_pitch;
  float best;
  const int bi = warp_argmax_first(nc, [&](int k) { return sigmoid_fast(__ldg(c + k)); }, best);
  if (lane == 0) {
    const float* r = ro + (size_t)warp * ro_pitch;
    const float cx = __fmul_rn(__fadd_rn(__ldg(r), (float)px), stride);
    const float cy = __fmul_rn(__fadd_rn(__ldg(r + 1), (float)py), stride);
    const float w = __fmul_rn(expf(__ldg(r + 2)), stride);
    const float h = __fmul_rn(expf(__ldg(r + 3)), stride);
    const float obj = sigmoid_fast(__ldg(r + 4));
    const float hw2 = __fdiv_rn(w, 2.0f), hh2 = __fdiv_rn(h, 2.0f);
    float4* o = reinterpret_cast<float4*>(cand + ((size_t)b * A + off + p) * 8);
    o[0] = make_float4(__fsub_rn(cx, hw2), __fsub_rn(cy, hh2), __fadd_rn(cx, hw2), __fadd_rn(cy, hh2));
    o[1] = make_float4(obj, best, (float)bi, __fmul_rn(obj, best));
  }
}

constexpr int kXThreads = 1024;
constexpr int kXKeys = 16384;   // candidate capacity per image (head locations; 8972 at 640x640)
constexpr int kXChunk = 512;

struct YoloxSmem {
  uint64_t keys[kXKeys];
  GreedyChunk<kXChunk> g;  // boxes as seen by NMS (class offset added in coordinate-trick mode); payload = candidate index
  float red[kXThreads / 32];
  int cls_head[1024];      // per-class (hashed by class & 1023) chain of kept boxes: head index, links in knext (-1 = end)
  uint32_t n;
};

// One CTA per image: score filter (obj * class_conf >= conf_thre, :58), stable descending order (score, then lower index),
// torchvision.ops.batched_nms: more than `vanilla_above` boxes -> per-class NMS on the raw boxes (_batched_nms_vanilla),
// else one NMS on boxes + class * (max_coordinate + 1) (_batched_nms_coordinate_trick); IoU in fp32, compared in double,
// areas without +1.  Rows (x1, y1, x2, y2, obj, class_conf, class_pred) are written in kept (score) order.
__global__ void __launch_bounds__(kXThreads) yolox_nms_kernel(const float* __restrict__ cand, int A, float conf, double iou_thr,
                                                              int vanilla_above, float* __restrict__ det, int* __restrict__ count,
                                                              float4* __restrict__ kbox_g, float* __restrict__ karea_g, int* __restrict__ kcls_g,
                                                              int* __restrict__ knext_g) {
  extern __shared__ uint8_t xs_raw[];
  YoloxSmem& S = *reinterpret_cast<YoloxSmem*>(xs_raw);
  const int b = blockIdx.x;
  const int tid = threadIdx.x;
  const float* cb = cand + (size_t)b * A * 8;
  float4* kbox = kbox_g + (size_t)b * A;
  float* karea = karea_g + (size_t)b * A;
  int* kcls = kcls_g + (size_t)b * A;
  int* knext = knext_g + (size_t)b * A;
  float* dout = det + (size_t)b * A * 7;
  if (tid == 0) S.n = 0;
  for (int i = tid; i < 1024; i += kXThreads) S.cls_head[i] = -1;
  __syncthreads();
  float cmax = -CUDART_INF_F;
  for (int i = tid; i < A; i += kXThreads) {
    const float4 hi = __ldg(reinterpret_cast<const float4*>(cb + (size_t)i * 8 + 4));
    if (hi.w >= conf) {
      const float4 bx = __ldg(reinterpret_cast<const float4*>(cb + (size_t)i * 8));
      cmax = fmaxf(cmax, fmaxf(fmaxf(bx.x, bx.y), fmaxf(bx.z, bx.w)));
      S.keys[atomicAdd(&S.n, 1u)] = make_key(__float_as_uint(hi.w), (uint32_t)i);
    }
  }
  // max_coordinate + 1 (torchvision/ops/boxes.py _batched_nms_coordinate_trick)
  const float unit = __fadd_rn(block_max<kXThreads>(cmax, S.red), 1.0f);
  const int n = (int)S.n;
  if (n == 0) {
    if (tid == 0) count[b] = 0;
    return;
  }
  int npad = 1;
  while (npad < n) npad <<= 1;
  for (int i = n + tid; i < npad; i += kXThreads) S.keys[i] = 0ull;
  bitonic_tile(S.keys, npad, 0, 2, npad);
  __syncthreads();
  const bool vanilla = n > vanilla_above;
  int kept_n = 0;
  for (int base = 0; base < n; base += kXChunk) {
    const int i = base + tid;
    bool alive = tid < kXChunk && i < n;
    float4 box = make_float4(0, 0, 0, 0);
    float area = 0.0f;
    int cls = 0;
    uint32_t idx = 0;
    if (alive) {
      idx = key_id(S.keys[i]);
      const float4 bx = __ldg(reinterpret_cast<const float4*>(cb + (size_t)idx * 8));
      const float4 hi = __ldg(reinterpret_cast<const float4*>(cb + (size_t)idx * 8 + 4));
      cls = (int)hi.z;
      if (vanilla) {
        box = bx;
      } else {
        const float offv = __fmul_rn((float)cls, unit);
        box = make_float4(__fadd_rn(bx.x, offv), __fadd_rn(bx.y, offv), __fadd_rn(bx.z, offv), __fadd_rn(bx.w, offv));
      }
      area = __fmul_rn(__fsub_rn(box.z, box.x), __fsub_rn(box.w, box.y));
      if (vanilla) {
        // class-wise NMS: only kept boxes of the same class can suppress -> walk that class's chain (any order)
        for (int k = S.cls_head[cls & 1023]; k >= 0; k = knext[k]) {
          if (kcls[k] == cls && iou_gt(kbox[k], karea[k], box, area, iou_thr)) {
            alive = false;
            break;
          }
        }
      } else {
        for (int k = 0; k < kept_n; ++k) {
          if (iou_gt(kbox[k], karea[k], box, area, iou_thr)) {
            alive = false;
            break;
          }
        }
      }
    }
    const int nk = greedy_chunk<kXThreads>(S.g, alive, box, area, cls, idx, kXChunk,
                                           [&](int r, int c) {
                                             const GreedyChunk<kXChunk>& G = S.g;
                                             return (!vanilla || G.cls[c] == G.cls[r]) && iou_gt(G.box[r], G.area[r], G.box[c], G.area[c], iou_thr);
                                           });
    for (int t = tid; t < nk; t += kXThreads) {
      const int r = (int)S.g.keep[t];
      const int o = kept_n + t;
      kbox[o] = S.g.box[r];
      karea[o] = S.g.area[r];
      kcls[o] = S.g.cls[r];
      knext[o] = atomicExch(&S.cls_head[S.g.cls[r] & 1023], o);
      const float* src = cb + (size_t)S.g.payload[r] * 8;
      float* d = dout + (size_t)o * 7;
#pragma unroll
      for (int q = 0; q < 7; ++q) d[q] = __ldg(src + q);
    }
    kept_n += nk;
    __threadfence_block();
    __syncthreads();
  }
  if (tid == 0) count[b] = kept_n;
}

}  // namespace cvb

extern "C" size_t cvb_yolox_workspace_bytes(int32_t B, int32_t A) {
  if (B <= 0 || A <= 0) return 0;
  return (size_t)B * A * (sizeof(float4) + sizeof(float) + 2 * sizeof(int));
}

extern "C" int cvb_yolox_decode(const CvbView* reg_obj, const CvbView* cls, int32_t nc, float stride, float* cand, int64_t A, int64_t off,
                                void* stream) {
  using namespace cvb;
  CVB_REQUIRE(reg_obj && cls && reg_obj->base && cls->base && cand, "yolox_decode: null argument");
  CVB_REQUIRE(reg_obj->plane_stride == 0 && cls->plane_stride == 0, "yolox_decode: inputs must be fp32 NHWC views");
  CVB_REQUIRE(reg_obj->B == cls->B && reg_obj->H == cls->H && reg_obj->W == cls->W && reg_obj->C >= 5 && cls->C >= nc && nc > 0,
              "yolox_decode: shape mismatch");
  CVB_REQUIRE(off >= 0 && off + (int64_t)cls->H * cls->W <= A && is_aligned(cand, 16), "yolox_decode: bad output range");
  const long long npix = (long long)cls->B * cls->H * cls->W;
  const long long blocks = (npix * 32 + 255) / 256;
  yolox_decode_kernel<<<(unsigned)blocks, 256, 0, as_stream(stream)>>>(static_cast<const float*>(reg_obj->base), reg_obj->c_pitch,
                                                                        static_cast<const float*>(cls->base), cls->c_pitch, cls->B, cls->H, cls->W, nc,
                                                                        stride, cand, A, off);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}

extern "C" int cvb_yolox_nms(const float* cand, int32_t B, int32_t A, float conf_thres, double iou_thres, int32_t vanilla_above, float* det,
                             int32_t* det_count, void* workspace, size_t workspace_bytes, void* stream) {
  using namespace cvb;
  CVB_REQUIRE(cand && det && det_count && workspace && B > 0 && A > 0, "yolox_nms: null argument / bad shape");
  CVB_REQUIRE(A <= kXKeys, "yolox_nms: at most %d locations per image (got %d)", kXKeys, A);
  CVB_REQUIRE(workspace_bytes >= cvb_yolox_workspace_bytes(B, A) && is_aligned(workspace, 16), "yolox_nms: workspace");
  CVB_REQUIRE(is_aligned(cand, 16), "yolox_nms: candidate records must be 16-byte aligned");
  // one-time, thread-safe (C++11 static initialisation) opt-in to the large dynamic shared memory carve-out
  static const cudaError_t attr_set_err = opt_in_smem(yolox_nms_kernel, (int)sizeof(YoloxSmem));
  CVB_CHECK_CUDA(attr_set_err);
  float4* kbox = static_cast<float4*>(workspace);
  float* karea = reinterpret_cast<float*>(kbox + (size_t)B * A);
  int* kcls = reinterpret_cast<int*>(karea + (size_t)B * A);
  int* knext = kcls + (size_t)B * A;
  yolox_nms_kernel<<<B, kXThreads, sizeof(YoloxSmem), as_stream(stream)>>>(cand, A, conf_thres, iou_thres, vanilla_above, det, det_count, kbox, karea,
                                                                          kcls, knext);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}

// =====================================================================================================================
// FCOS post-processing (src/models/detects/fcos_detect.py:42-153)
// =====================================================================================================================
namespace cvb {

// One warp per location: max over class sigmoids (first maximum wins), score = sqrt(cls * sigmoid(cnt)), class id + 1,
// box = (cx - l, cy - t, cx + r, cy + b) with ltrb = exp(raw * scale_i) (ScaleExp, fcos_head.py:13-19) and the location
// centre (x*stride + stride//2, y*stride + stride//2) (coords_fmap2orig :14-31).
__global__ void __launch_bounds__(256) fcos_decode_kernel(const float* __restrict__ cls, int cls_pitch, const float* __restrict__ rc,
                                                          int rc_pitch, int B, int h, int w, int nc, float stride, float scale,
                                                          float* __restrict__ scores, int* __restrict__ classes,
                                                          float* __restrict__ boxes, long long n_total, long long loc_off) {
  const int lane = threadIdx.x & 31;
  const long long npix = (long long)h * w;
  const long long rows = (long long)B * npix;
  const long long wstride = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long row = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5); row < rows; row += wstride) {
    const int b = (int)(row / npix);
    const int pix = (int)(row - (long long)b * npix);
    const float* c = cls + row * cls_pitch;
    float best;
    const int bi = warp_argmax_first(nc, [&](int k) { return sigmoid_fast(__ldg(c + k)); }, best);
    if (lane == 0) {
      const float* r = rc + row * rc_pitch;
      const float cnt = sigmoid_fast(__ldg(r + 4));
      const int py = pix / w, px = pix - py * w;
      const float half = (float)(((int)stride) / 2);
      const float cx = __fadd_rn(__fmul_rn((float)px, stride), half), cy = __fadd_rn(__fmul_rn((float)py, stride), half);
      const float l = expf(__fmul_rn(__ldg(r + 0), scale)), t = expf(__fmul_rn(__ldg(r + 1), scale));
      const float rr = expf(__fmul_rn(__ldg(r + 2), scale)), bb = expf(__fmul_rn(__ldg(r + 3), scale));
      const size_t o = (size_t)b * n_total + loc_off + pix;
      scores[o] = sqrtf(__fmul_rn(best, cnt));
      classes[o] = bi + 1;
      float4 bx = make_float4(__fsub_rn(cx, l), __fsub_rn(cy, t), __fadd_rn(cx, rr), __fadd_rn(cy, bb));
      *reinterpret_cast<float4*>(boxes + o * 4) = bx;
    }
  }
}

constexpr int kFcosThreads = 512;
constexpr int kFcosSel = 4096;  // candidates sorted in shared memory (top-k <= 2048 supported)

struct FcosSmem {
  uint64_t keys[kFcosSel];                 // 32 KB
  union {
    uint32_t hist[kBins];                  // 64 KB, top-k selection
    GreedyChunk<kFcosThreads> g;           // greedy scan, after the selection; payload = sorted key position
  };
  float4 kbox[2048];                       // kept (class-offset) boxes, 32 KB
  float karea[2048];
  uint32_t seg[kBins / 32];
  uint32_t warp_cnt[kFcosThreads / 32];
  float red[kFcosThreads / 32];
  uint32_t n_sel, tbin, overflow;
};

// FCOS IoU: '+1' areas, plain intersection, box j is KEPT iff iou <= thr evaluated in float32 (fcos_detect.py:117,133-135)
__device__ __forceinline__ bool fcos_suppressed(const float4& a, float aa, const float4& b, float ab, float thr32) {
  const float xmin = fmaxf(b.x, a.x), ymin = fmaxf(b.y, a.y);
  const float xmax = fminf(b.z, a.z), ymax = fminf(b.w, a.w);
  const float inter = __fmul_rn(fmaxf(__fsub_rn(xmax, xmin), 0.0f), fmaxf(__fsub_rn(ymax, ymin), 0.0f));
  const float iou = __fdiv_rn(inter, __fsub_rn(__fadd_rn(aa, ab), inter));
  return !(iou <= thr32);
}

// Score as the top-k selection sees it.  -0.0f equals 0 (torch.topk and the score threshold treat it so), but its bit pattern would
// land in the top histogram bin and sort above every positive score: it is selected as +0.0f.
__device__ __forceinline__ float fcos_score(float v) { return v == 0.0f ? 0.0f : v; }

__global__ void __launch_bounds__(kFcosThreads) fcos_nms_kernel(const float* __restrict__ scores, const int* __restrict__ classes,
                                                                const float* __restrict__ boxes, int N, float score_thres,
                                                                float iou_thres, int topk, float* __restrict__ out_scores,
                                                                int* __restrict__ out_classes, float* __restrict__ out_boxes,
                                                                int* __restrict__ out_loc, int* __restrict__ out_count,
                                                                int* __restrict__ status) {
  extern __shared__ uint8_t fs_raw[];
  FcosSmem& S = *reinterpret_cast<FcosSmem*>(fs_raw);
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* sc = scores + (size_t)b * N;
  const int* cl = classes + (size_t)b * N;
  const float4* bx = reinterpret_cast<const float4*>(boxes) + (size_t)b * N;

  // ---- 1. top-k selection: histogram of score bits -> threshold bin -> collect -> bitonic sort (descending; ties: lower index)
  for (int i = tid; i < kBins; i += kFcosThreads) S.hist[i] = 0;
  if (tid == 0) {
    S.n_sel = 0;
    S.overflow = 0;
  }
  __syncthreads();
  for (int i = tid; i < N; i += kFcosThreads) {
    const float v = fcos_score(sc[i]);
    if (v >= 0.0f) atomicAdd(&S.hist[nms_score_bin(v)], 1u);  // NaN / negative never selected
  }
  __syncthreads();
  top_bin_search<kFcosThreads>(S.hist, (uint32_t)topk, S.seg, &S.tbin, nullptr);
  __syncthreads();
  const uint32_t tb = S.tbin;
  for (int i0 = 0; i0 < N; i0 += kFcosThreads) {
    const int i = i0 + tid;
    const float v = (i < N) ? fcos_score(sc[i]) : 0.0f;
    const bool pass = i < N && v >= 0.0f && nms_score_bin(v) >= tb;
    const uint32_t pos = warp_append(&S.n_sel, pass);
    if (pass) {
      if (pos < (uint32_t)kFcosSel) S.keys[pos] = make_key(__float_as_uint(v), (uint32_t)i);
      else S.overflow = 1;
    }
  }
  __syncthreads();
  uint32_t nsel = min(S.n_sel, (uint32_t)kFcosSel);
  if (S.overflow && status && tid == 0) atomicExch(&status[0], 1);
  for (int i = nsel + tid; i < kFcosSel; i += kFcosThreads) S.keys[i] = 0ull;
  bitonic_tile(S.keys, kFcosSel, 0, 2, kFcosSel);
  __syncthreads();
  // candidates = sorted prefix of length min(topk, nsel) with score >= score_thres (fcos_detect.py:65-67,92-93)
  int ncand = min((int)nsel, topk);
  {
    // scores are sorted descending: count the prefix that passes the threshold
    int cntp = 0;
    for (int i = tid; i < ncand; i += kFcosThreads) cntp += (key_score(S.keys[i]) >= score_thres) ? 1 : 0;
    for (int o = 16; o > 0; o >>= 1) cntp += __shfl_xor_sync(0xffffffffu, cntp, o);
    if (lane == 0) S.warp_cnt[warp] = (uint32_t)cntp;
    __syncthreads();
    int tot = 0;
    for (int i = 0; i < kFcosThreads / 32; ++i) tot += (int)S.warp_cnt[i];
    ncand = tot;
    __syncthreads();
  }
  // ---- 2. class offset = cls * (max coordinate of the candidate boxes + 1)   (batched_nms :141-153)
  float mx = -3.402823466e38f;
  for (int i = tid; i < ncand; i += kFcosThreads) {
    const float4 q = bx[key_id(S.keys[i])];
    mx = fmaxf(mx, fmaxf(fmaxf(q.x, q.y), fmaxf(q.z, q.w)));
  }
  const float offmul = __fadd_rn(block_max<kFcosThreads>(mx, S.red), 1.0f);

  // ---- 3. greedy NMS over the candidates in score order (chunks of 512, like the YOLO kernel)
  int kept_n = 0;
  for (int base = 0; base < ncand; base += kFcosThreads) {
    const int i = base + tid;
    bool alive = i < ncand;
    float4 box = make_float4(0, 0, 0, 0);
    float area = 0.0f;
    if (alive) {
      const uint32_t loc = key_id(S.keys[i]);
      const float4 q = bx[loc];
      const float off = __fmul_rn((float)cl[loc], offmul);
      box = make_float4(__fadd_rn(q.x, off), __fadd_rn(q.y, off), __fadd_rn(q.z, off), __fadd_rn(q.w, off));
      area = __fmul_rn(__fadd_rn(__fsub_rn(box.z, box.x), 1.0f), __fadd_rn(__fsub_rn(box.w, box.y), 1.0f));
      for (int k = 0; k < kept_n; ++k)
        if (fcos_suppressed(S.kbox[k], S.karea[k], box, area, iou_thres)) {
          alive = false;
          break;
        }
    }
    const int nk = greedy_chunk<kFcosThreads>(S.g, alive, box, area, 0, (uint32_t)i, kFcosThreads,
                                              [&](int r, int c) {
                                                return fcos_suppressed(S.g.box[r], S.g.area[r], S.g.box[c], S.g.area[c], iou_thres);
                                              });
    for (int t = tid; t < nk; t += kFcosThreads) {
      const int r = (int)S.g.keep[t];
      const int o = kept_n + t;
      S.kbox[o] = S.g.box[r];
      S.karea[o] = S.g.area[r];
      const uint64_t key = S.keys[S.g.payload[r]];
      const uint32_t l2 = key_id(key);
      out_scores[(size_t)b * topk + o] = key_score(key);
      out_classes[(size_t)b * topk + o] = cl[l2];
      reinterpret_cast<float4*>(out_boxes)[(size_t)b * topk + o] = bx[l2];
      out_loc[(size_t)b * topk + o] = (int)l2;
    }
    kept_n += nk;
    __syncthreads();
  }
  if (tid == 0) out_count[b] = kept_n;
}

}  // namespace cvb

extern "C" int cvb_fcos_decode(const CvbView* cls, const CvbView* regcnt, int32_t nc, float stride, float scale, float* scores,
                               int32_t* classes, float* boxes, int64_t n_total, int64_t loc_off, void* stream) {
  using namespace cvb;
  CVB_REQUIRE(cls && regcnt && cls->base && regcnt->base && scores && classes && boxes, "fcos_decode: null argument");
  CVB_REQUIRE(cls->B == regcnt->B && cls->H == regcnt->H && cls->W == regcnt->W && cls->c_pitch >= nc && regcnt->c_pitch >= 5,
              "fcos_decode: view mismatch");
  CVB_REQUIRE(is_aligned(boxes, 16), "fcos_decode: boxes must be 16-byte aligned");
  const long long rows = (long long)cls->B * cls->H * cls->W;
  long long grid = (rows + 7) / 8;
  if (grid > kSmCount * 16) grid = kSmCount * 16;
  fcos_decode_kernel<<<(int)grid, 256, 0, as_stream(stream)>>>(static_cast<const float*>(cls->base), cls->c_pitch,
                                                              static_cast<const float*>(regcnt->base), regcnt->c_pitch, cls->B, cls->H,
                                                              cls->W, nc, stride, scale, scores, classes, boxes, n_total, loc_off);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}

extern "C" int cvb_fcos_nms(const float* scores, const int32_t* classes, const float* boxes, int32_t B, int32_t N, float score_thres,
                            float iou_thres, int32_t topk, float* out_scores, int32_t* out_classes, float* out_boxes, int32_t* out_loc,
                            int32_t* out_count, int32_t* status, void* stream) {
  using namespace cvb;
  CVB_REQUIRE(scores && classes && boxes && out_scores && out_classes && out_boxes && out_loc && out_count, "fcos_nms: null argument");
  CVB_REQUIRE(B > 0 && N > 0 && topk > 0 && topk <= 2048, "fcos_nms: bad sizes (topk <= 2048)");
  CVB_REQUIRE(is_aligned(boxes, 16) && is_aligned(out_boxes, 16), "fcos_nms: box arrays must be 16-byte aligned");
  cudaStream_t st = as_stream(stream);
  if (status) CVB_CHECK_CUDA(cudaMemsetAsync(status, 0, 4 * sizeof(int32_t), st));
  CVB_CHECK_CUDA(cudaMemsetAsync(out_scores, 0, (size_t)B * topk * sizeof(float), st));
  CVB_CHECK_CUDA(cudaMemsetAsync(out_classes, 0, (size_t)B * topk * sizeof(int32_t), st));
  CVB_CHECK_CUDA(cudaMemsetAsync(out_boxes, 0, (size_t)B * topk * 4 * sizeof(float), st));
  CVB_CHECK_CUDA(cudaMemsetAsync(out_loc, 0xFF, (size_t)B * topk * sizeof(int32_t), st));
  // one-time, thread-safe (C++11 static initialisation) opt-in to the large dynamic shared memory carve-out
  static const cudaError_t attr_set_err = opt_in_smem(fcos_nms_kernel, (int)sizeof(FcosSmem));
  CVB_CHECK_CUDA(attr_set_err);
  fcos_nms_kernel<<<B, kFcosThreads, sizeof(FcosSmem), st>>>(scores, classes, boxes, N, score_thres, iou_thres, topk, out_scores, out_classes,
                                                            out_boxes, out_loc, out_count, status);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}
