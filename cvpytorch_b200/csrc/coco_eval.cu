// COCO box mAP on the device (pycocotools COCOeval, iouType 'bbox', default parameters): the same matches, and precision / recall
// arrays equal bit for bit.  Stream-ordered, no host sync; the caller reads the 12 statistics with one 96-byte copy.
//
// 1. Group.   key1 = (category * n_images + image) << 32 | descending-score bits, radix-sorted stably, so every (category, image) segment
//             lists its detections by -score with ties in input order (COCOeval's mergesort).  Detections of no evaluated category get
//             an all-ones key and sort last.  Segment heads are selected with CUB.
// 2. Match.   One CTA per segment (grid-stride).  Threads 0..39 are the 4 area ranges x 10 IoU thresholds, each an independent greedy
//             scan over the segment's first 100 detections.  The IoU tile (detections x kGtTile ground truths) lives in shared memory
//             in float64; a segment with more ground truths than one tile recomputes one detection's row per tile.  The ignore-sorted
//             GT order of COCOeval is never built: the scan keeps the best candidate among the non-ignored ground truths and among the
//             ignored ones (max IoU >= bound, the last one on ties) and takes the ignored candidate only when no non-ignored one
//             matched, which is what the sorted scan with its early break computes.  Output: per detection and area range a 10-bit
//             matched mask (bits 0..9) and a 10-bit ignored mask (bits 16..25).
// 3. Count.   Non-ignored ground truths per (category, area range) over the evaluated images, integer atomics.
// 4. Accumulate.  key2 = category << 32 | descending-score bits for the kept detections (rank < 100), stably sorted after step 1's
//             order, so ties fall back to ascending image id, then rank.  One CTA per (category, area, maxDet) walks the category's
//             detections backwards per threshold: block scans give tp / fp prefix counts and the suffix maximum of the precision,
//             and each detection whose recall rises assigns the recall thresholds it crosses (searchsorted 'left' seen from rc's side).
// 5. Summarize.  One CTA per statistic: the mean of the entries > -1 of its slice in float64, summed in a fixed order.
//
// Built with --fmad=false: the IoU's (da + ga) - w * h and the precision's tp / ((tp + fp) + eps) must round like the host's.
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_select.cuh>

#include <algorithm>

#include "internal.h"

namespace cvb {

constexpr int kCocoT = CVB_COCO_IOU_THRS, kCocoR = CVB_COCO_REC_THRS, kCocoA = 4, kCocoM = 3;
constexpr int kCocoMaxDet = 100;
constexpr int kScans = kCocoA * kCocoT;  // 40 greedy scans per segment
constexpr int kMatchThreads = 64;
constexpr int kGtTile = 32;
constexpr int kAccThreads = 256;
constexpr int kSumThreads = 256;
constexpr uint64_t kDropKey = ~0ull;
constexpr uint32_t kDropSeg = 0xFFFFFFFFu;

__constant__ double kAreaLo[kCocoA] = {0.0, 0.0, 1024.0, 9216.0};
__constant__ double kAreaHi[kCocoA] = {1e10, 1024.0, 9216.0, 1e10};
__constant__ int kMaxDets[kCocoM] = {1, 10, 100};

// descending-score radix key: -0.0 is +0.0 (COCOeval compares -score), NaN never reaches the device
__device__ __forceinline__ uint32_t score_desc_key(float s) {
  const uint32_t b = __float_as_uint(s == 0.f ? 0.f : s);
  return ~((b & 0x80000000u) ? ~b : (b | 0x80000000u));
}

template <typename T>
__device__ __forceinline__ int lower_bound(const T* a, int n, T v) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (a[mid] < v) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// maskApi.c bbIou: xywh boxes in float64, crowd ground truths divide by the detection area
__device__ __forceinline__ double bb_iou(const double* d, double da, const double* g, bool crowd) {
  const double w = __dsub_rn(fmin(__dadd_rn(d[0], d[2]), __dadd_rn(g[0], g[2])), fmax(d[0], g[0]));
  if (w <= 0) return 0.0;
  const double h = __dsub_rn(fmin(__dadd_rn(d[1], d[3]), __dadd_rn(g[1], g[3])), fmax(d[1], g[1]));
  if (h <= 0) return 0.0;
  const double i = __dmul_rn(w, h);
  const double u = crowd ? da : __dsub_rn(__dadd_rn(da, __dmul_rn(g[2], g[3])), i);
  return __ddiv_rn(i, u);
}

__global__ void coco_keys_kernel(int n, int n_images, const int32_t* __restrict__ det_img, const int32_t* __restrict__ det_cat,
                                 const float* __restrict__ det_score, uint64_t* __restrict__ keys, int32_t* __restrict__ vals) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c = det_cat[i];
  keys[i] = c < 0 ? kDropKey : ((uint64_t)((uint32_t)c * (uint32_t)n_images + (uint32_t)det_img[i]) << 32) | score_desc_key(det_score[i]);
  vals[i] = i;
}

__global__ void coco_heads_kernel(int n, const uint64_t* __restrict__ keys, uint8_t* __restrict__ flags, int32_t* __restrict__ idx) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  flags[i] = i == 0 || (keys[i] >> 32) != (keys[i - 1] >> 32);
  idx[i] = i;
}

__global__ void __launch_bounds__(kMatchThreads) coco_match_kernel(CvbCocoEvalParams p, const uint64_t* __restrict__ keys,
    const int32_t* __restrict__ order, const int32_t* __restrict__ seg_start, const int32_t* __restrict__ num_segs,
    const uint32_t* __restrict__ gt_key, const double* __restrict__ gt_box, const double* __restrict__ gt_area,
    const uint8_t* __restrict__ gt_crowd, const double* __restrict__ det_box, uint8_t* __restrict__ gt_matched,
    uint64_t* __restrict__ key2, int32_t* __restrict__ det_rank, uint32_t* __restrict__ det_masks) {
  __shared__ double s_iou[kCocoMaxDet][kGtTile];
  __shared__ double s_dbox[kCocoMaxDet][4];
  __shared__ double s_darea[kCocoMaxDet];
  __shared__ double s_gbox[kGtTile][4];
  __shared__ double s_garea[kGtTile];
  __shared__ uint8_t s_gcrowd[kGtTile];
  __shared__ uint32_t s_mask[kCocoMaxDet][kCocoA];
  const int tid = threadIdx.x;
  const int t = tid % kCocoT, a = tid / kCocoT;
  const double thr0 = tid < kScans ? fmin(p.iou_thrs[t], 1 - 1e-10) : 0.0;
  const double alo = tid < kScans ? kAreaLo[a] : 0.0, ahi = tid < kScans ? kAreaHi[a] : 0.0;
  const int nseg = *num_segs;
  for (int s = blockIdx.x; s < nseg; s += gridDim.x) {
    const int p0 = seg_start[s], p1 = s + 1 < nseg ? seg_start[s + 1] : p.n_det;
    const uint32_t seg = (uint32_t)(keys[p0] >> 32);
    if (seg == kDropSeg) {
      for (int q = p0 + tid; q < p1; q += kMatchThreads) key2[q] = kDropKey;
      continue;
    }
    const uint32_t cat = seg / (uint32_t)p.n_images;
    for (int q = p0 + tid; q < p1; q += kMatchThreads) {
      const int r = q - p0;
      det_rank[order[q]] = r;
      key2[q] = r < kCocoMaxDet ? ((uint64_t)cat << 32) | (uint32_t)keys[q] : kDropKey;
    }
    const int D = min(p1 - p0, kCocoMaxDet);
    const int g0 = lower_bound(gt_key, p.n_gt, seg), g1 = lower_bound(gt_key, p.n_gt, seg + 1);
    const int G = g1 - g0, nt = (G + kGtTile - 1) / kGtTile;
    __syncthreads();  // the previous segment is done with the shared tiles
    for (int d = tid; d < D; d += kMatchThreads) {
      const double* b = det_box + (int64_t)order[p0 + d] * 4;
      for (int c = 0; c < 4; ++c) s_dbox[d][c] = b[c];
      s_darea[d] = __dmul_rn(b[2], b[3]);
      for (int c = 0; c < kCocoA; ++c) s_mask[d][c] = 0;
    }
    __syncthreads();
    for (int d = 0; d < D; ++d) {
      double best_n = thr0, best_i = thr0;  // best non-ignored / ignored candidate so far
      int m_n = -1, m_i = -1;
      for (int j = 0; j < nt; ++j) {
        const int cols = min(kGtTile, G - j * kGtTile);
        if (nt > 1 || d == 0) {  // one tile holds every ground truth: fill it once; otherwise one detection row per tile
          __syncthreads();
          const int rows = nt > 1 ? 1 : D, row0 = nt > 1 ? d : 0;
          for (int e = tid; e < cols; e += kMatchThreads) {
            const int g = g0 + j * kGtTile + e;
            for (int c = 0; c < 4; ++c) s_gbox[e][c] = gt_box[(int64_t)g * 4 + c];
            s_garea[e] = gt_area[g];
            s_gcrowd[e] = gt_crowd[g];
          }
          __syncthreads();
          for (int e = tid; e < rows * cols; e += kMatchThreads) {
            const int r = e / cols, c = e % cols;
            s_iou[r][c] = bb_iou(s_dbox[row0 + r], s_darea[row0 + r], s_gbox[c], s_gcrowd[c] != 0);
          }
          __syncthreads();
        }
        if (tid < kScans) {
          const int row = nt > 1 ? 0 : d;
          for (int c = 0; c < cols; ++c) {
            const int g = g0 + j * kGtTile + c;
            const bool crowd = s_gcrowd[c] != 0;
            if (!crowd && gt_matched[(int64_t)g * kScans + tid]) continue;
            const double v = s_iou[row][c];
            if (crowd || s_garea[c] < alo || s_garea[c] > ahi) {
              if (v >= best_i) best_i = v, m_i = g;
            } else if (v >= best_n) {
              best_n = v, m_n = g;
            }
          }
        }
      }
      if (tid < kScans) {
        const int m = m_n >= 0 ? m_n : m_i;
        uint32_t bits;
        if (m >= 0) {
          gt_matched[(int64_t)m * kScans + tid] = 1;
          bits = (1u << t) | (m_n < 0 ? 1u << (16 + t) : 0u);
        } else {
          bits = (s_darea[d] < alo || s_darea[d] > ahi) ? 1u << (16 + t) : 0u;
        }
        atomicOr(&s_mask[d][a], bits);
      }
    }
    __syncthreads();
    for (int e = tid; e < D * kCocoA; e += kMatchThreads) det_masks[(int64_t)order[p0 + e / kCocoA] * kCocoA + e % kCocoA] = s_mask[e / kCocoA][e % kCocoA];
  }
}

__global__ void coco_npig_kernel(CvbCocoEvalParams p, const uint32_t* __restrict__ gt_key, const double* __restrict__ gt_area,
                                 const uint8_t* __restrict__ gt_crowd, const uint8_t* __restrict__ img_evaluated, int32_t* __restrict__ npig) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= p.n_gt) return;
  const uint32_t seg = gt_key[g];
  if (!img_evaluated[seg % (uint32_t)p.n_images] || gt_crowd[g]) return;
  const int k = seg / (uint32_t)p.n_images;
  for (int a = 0; a < kCocoA; ++a)
    if (!(gt_area[g] < kAreaLo[a] || gt_area[g] > kAreaHi[a])) atomicAdd(&npig[k * kCocoA + a], 1);
}

struct MaxOp {
  __device__ __forceinline__ double operator()(double x, double y) const { return fmax(x, y); }
};

__global__ void __launch_bounds__(kAccThreads) coco_accumulate_kernel(CvbCocoEvalParams p, const uint64_t* __restrict__ key2,
    const int32_t* __restrict__ order2, const int32_t* __restrict__ det_rank, const uint32_t* __restrict__ det_masks,
    const int32_t* __restrict__ npig_all, double* __restrict__ precision, double* __restrict__ recall) {
  using Scan = cub::BlockScan<unsigned long long, kAccThreads>;
  using MaxScan = cub::BlockScan<double, kAccThreads>;
  using Reduce = cub::BlockReduce<unsigned long long, kAccThreads>;
  __shared__ union {
    typename Scan::TempStorage scan;
    typename MaxScan::TempStorage max_scan;
    typename Reduce::TempStorage reduce;
  } tmp;
  __shared__ double s_q[kCocoR];
  __shared__ unsigned long long s_total;
  const int k = blockIdx.x / (kCocoA * kCocoM), a = blockIdx.x / kCocoM % kCocoA, m = blockIdx.x % kCocoM;
  const int K = p.n_cats, tid = threadIdx.x;
  const int npig = npig_all[k * kCocoA + a];
  auto pidx = [&](int t, int r) { return ((((int64_t)t * kCocoR + r) * K + k) * kCocoA + a) * kCocoM + m; };
  if (npig == 0) {
    for (int e = tid; e < kCocoT * kCocoR; e += kAccThreads) precision[pidx(e / kCocoR, e % kCocoR)] = -1.0;
    if (tid < kCocoT) recall[(((int64_t)tid * K + k) * kCocoA + a) * kCocoM + m] = -1.0;
    return;
  }
  const int lo = lower_bound(key2, p.n_det, (uint64_t)k << 32), hi = lower_bound(key2, p.n_det, (uint64_t)(k + 1) << 32);
  const int max_det = kMaxDets[m];
  const double dn = (double)npig, eps = 2.220446049250313e-16;  // np.spacing(1)
  // tp in the high word, fp in the low word of a detection's count pair for threshold t (0 when beyond maxDet)
  auto pair = [&](int i, int t) -> unsigned long long {
    const int o = order2[i];
    if (det_rank[o] >= max_det) return 0ull;
    const uint32_t w = det_masks[(int64_t)o * kCocoA + a];
    if ((w >> (16 + t)) & 1u) return 0ull;
    return ((w >> t) & 1u) ? 1ull << 32 : 1ull;
  };
  for (int t = 0; t < kCocoT; ++t) {
    unsigned long long part = 0;
    for (int i = lo + tid; i < hi; i += kAccThreads) part += pair(i, t);
    const unsigned long long total = Reduce(tmp.reduce).Sum(part);
    if (tid == 0) s_total = total;
    for (int r = tid; r < kCocoR; r += kAccThreads) s_q[r] = 0.0;
    __syncthreads();
    const unsigned long long tot = s_total;
    unsigned long long carry = 0;  // counts of the detections after the current chunk
    double carry_env = 0.0;        // precision envelope (suffix maximum) of the detections after the current chunk
    for (int base = hi; base > lo; base -= kAccThreads) {
      const int i = base - 1 - tid;  // thread order runs backwards through the detections
      const bool valid = i >= lo;
      const unsigned long long v = valid ? pair(i, t) : 0ull;
      unsigned long long incl, agg;
      Scan(tmp.scan).InclusiveSum(v, incl, agg);
      __syncthreads();
      const unsigned long long cum = tot - (carry + incl) + v;  // counts of the detections up to and including i
      const double tp = (double)(uint32_t)(cum >> 32), fp = (double)(uint32_t)cum;
      const double rc = __ddiv_rn(tp, dn);
      const double pr = valid ? __ddiv_rn(tp, __dadd_rn(__dadd_rn(fp, tp), eps)) : 0.0;
      double env, env_agg;
      MaxScan(tmp.max_scan).InclusiveScan(pr, env, MaxOp(), env_agg);
      __syncthreads();
      env = fmax(env, carry_env);
      if (valid) {
        // recall thresholds r with rc[i-1] < r <= rc[i] (every r <= rc[i] for the first detection) land on this detection
        const double rc_prev = i == lo ? -1.0 : __ddiv_rn(tp - (double)(v >> 32), dn);
        if (i == lo || rc_prev < rc) {
          int r0 = 0, r1 = kCocoR;
          if (i != lo) {
            int l = 0, h = kCocoR;
            while (l < h) { const int mid = (l + h) >> 1; if (p.rec_thrs[mid] > rc_prev) h = mid; else l = mid + 1; }
            r0 = l;
          }
          int l = r0, h = kCocoR;
          while (l < h) { const int mid = (l + h) >> 1; if (p.rec_thrs[mid] > rc) h = mid; else l = mid + 1; }
          r1 = l;
          for (int r = r0; r < r1; ++r) s_q[r] = env;
        }
      }
      carry += agg;
      carry_env = fmax(carry_env, env_agg);
    }
    __syncthreads();
    for (int r = tid; r < kCocoR; r += kAccThreads) precision[pidx(t, r)] = s_q[r];
    if (tid == 0) recall[(((int64_t)t * K + k) * kCocoA + a) * kCocoM + m] = __ddiv_rn((double)(uint32_t)(tot >> 32), dn);
    __syncthreads();
  }
}

// statistic -> (is AP, IoU threshold index or -1 for all, area range, maxDet index), COCOeval.summarize's order
__constant__ int kStatSpec[12][4] = {{1, -1, 0, 2}, {1, 0, 0, 2}, {1, 5, 0, 2}, {1, -1, 1, 2}, {1, -1, 2, 2}, {1, -1, 3, 2},
                                     {0, -1, 0, 0}, {0, -1, 0, 1}, {0, -1, 0, 2}, {0, -1, 1, 2}, {0, -1, 2, 2}, {0, -1, 3, 2}};

__global__ void __launch_bounds__(kSumThreads) coco_summarize_kernel(int K, const double* __restrict__ precision, const double* __restrict__ recall,
                                                                     double* __restrict__ stats) {
  __shared__ double s_sum[kSumThreads];
  __shared__ long long s_cnt[kSumThreads];
  const int* spec = kStatSpec[blockIdx.x];
  const bool ap = spec[0] != 0;
  const int t0 = spec[1] < 0 ? 0 : spec[1], nt = spec[1] < 0 ? kCocoT : 1, a = spec[2], m = spec[3];
  const int R = ap ? kCocoR : 1;
  const int64_t n = (int64_t)nt * R * K;
  double sum = 0.0;
  long long cnt = 0;
  for (int64_t e = threadIdx.x; e < n; e += kSumThreads) {
    const int k = (int)(e % K);
    const int64_t tr = e / K;
    const int t = t0 + (int)(tr / R), r = (int)(tr % R);
    const double v = ap ? precision[((((int64_t)t * kCocoR + r) * K + k) * kCocoA + a) * kCocoM + m]
                        : recall[(((int64_t)t * K + k) * kCocoA + a) * kCocoM + m];
    if (v > -1) sum = __dadd_rn(sum, v), ++cnt;
  }
  s_sum[threadIdx.x] = sum;
  s_cnt[threadIdx.x] = cnt;
  __syncthreads();
  for (int w = kSumThreads / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) {
      s_sum[threadIdx.x] = __dadd_rn(s_sum[threadIdx.x], s_sum[threadIdx.x + w]);
      s_cnt[threadIdx.x] += s_cnt[threadIdx.x + w];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) stats[blockIdx.x] = s_cnt[0] ? __ddiv_rn(s_sum[0], (double)s_cnt[0]) : -1.0;
}

// workspace carve-up; every piece 256-byte aligned
struct CocoWs {
  uint64_t *keys_in, *keys, *key2_in, *key2;
  int32_t *vals_in, *order, *order2, *seg_start, *num_segs, *det_rank, *npig;
  uint8_t *flags, *gt_matched;
  void* cub_tmp;
  size_t cub_bytes, total;
};

// CUB's temporary storage for the sorts and the segment-head selection; 0 when CUB cannot size it
static size_t cub_tmp_bytes(int n) {
  size_t a = 0, b = 0;
  if (cub::DeviceRadixSort::SortPairs(nullptr, a, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const int32_t*)nullptr, (int32_t*)nullptr, n) !=
          cudaSuccess ||
      cub::DeviceSelect::Flagged(nullptr, b, (const int32_t*)nullptr, (const uint8_t*)nullptr, (int32_t*)nullptr, (int32_t*)nullptr, n) !=
          cudaSuccess)
    return 0;
  return std::max<size_t>(std::max(a, b), 1);
}

static CocoWs coco_ws(void* base, int n_det, int n_gt, int n_cats) {
  WsCarver c(base);
  CocoWs w{};
  const size_t n = (size_t)n_det;
  w.keys_in = (uint64_t*)c.take(n * 8);
  w.keys = (uint64_t*)c.take(n * 8);
  w.key2_in = (uint64_t*)c.take(n * 8);
  w.key2 = (uint64_t*)c.take(n * 8);
  w.vals_in = (int32_t*)c.take(n * 4);
  w.order = (int32_t*)c.take(n * 4);
  w.order2 = (int32_t*)c.take(n * 4);
  w.seg_start = (int32_t*)c.take(n * 4);
  w.num_segs = (int32_t*)c.take(4);
  w.det_rank = (int32_t*)c.take(n * 4);
  w.npig = (int32_t*)c.take((size_t)n_cats * kCocoA * 4);
  w.flags = (uint8_t*)c.take(n);
  w.gt_matched = (uint8_t*)c.take((size_t)n_gt * kScans);
  w.cub_bytes = cub_tmp_bytes(n_det);
  w.cub_tmp = c.take(w.cub_bytes);
  w.total = w.cub_bytes ? c.bytes() : 0;
  return w;
}

static bool coco_sizes_ok(int32_t n_det, int32_t n_gt, int32_t n_cats) {
  return n_det >= 0 && n_det <= CVB_COCO_MAX_DETS && n_gt >= 0 && n_gt <= CVB_COCO_MAX_GT && n_cats >= 1 && n_cats <= CVB_COCO_MAX_CATS;
}

}  // namespace cvb

using namespace cvb;

extern "C" size_t cvb_coco_eval_workspace_bytes(int32_t n_det, int32_t n_gt, int32_t n_cats) {
  if (!coco_sizes_ok(n_det, n_gt, n_cats)) return 0;
  return coco_ws(nullptr, n_det, n_gt, n_cats).total;
}

extern "C" int cvb_coco_eval_bbox(const CvbCocoEvalParams* params, const uint32_t* gt_key, const double* gt_box, const double* gt_area,
                                  const uint8_t* gt_crowd, const uint8_t* img_evaluated, const int32_t* det_img, const int32_t* det_cat,
                                  const float* det_score, const double* det_box, uint32_t* det_masks, double* precision, double* recall,
                                  double* stats, void* workspace, size_t ws_bytes, void* stream) {
  CVB_REQUIRE(params, "coco_eval_bbox: null params");
  const CvbCocoEvalParams p = *params;
  CVB_REQUIRE(p.n_images >= 1 && p.n_images <= CVB_COCO_MAX_IMAGES, "coco_eval_bbox: n_images %d outside [1, %d]", p.n_images,
              CVB_COCO_MAX_IMAGES);
  CVB_REQUIRE(p.n_cats >= 1 && p.n_cats <= CVB_COCO_MAX_CATS, "coco_eval_bbox: n_cats %d outside [1, %d]", p.n_cats, CVB_COCO_MAX_CATS);
  CVB_REQUIRE(p.n_gt >= 0 && p.n_gt <= CVB_COCO_MAX_GT, "coco_eval_bbox: n_gt %d outside [0, %d]", p.n_gt, CVB_COCO_MAX_GT);
  CVB_REQUIRE(p.n_det >= 0 && p.n_det <= CVB_COCO_MAX_DETS, "coco_eval_bbox: n_det %d outside [0, %d]", p.n_det, CVB_COCO_MAX_DETS);
  CVB_REQUIRE(img_evaluated && precision && recall && stats && workspace, "coco_eval_bbox: null pointer");
  CVB_REQUIRE(p.n_gt == 0 || (gt_key && gt_box && gt_area && gt_crowd), "coco_eval_bbox: null ground-truth pointer");
  CVB_REQUIRE(p.n_det == 0 || (det_img && det_cat && det_score && det_box && det_masks), "coco_eval_bbox: null detection pointer");
  CVB_REQUIRE(is_aligned(workspace, 256), "coco_eval_bbox: workspace must be 256-byte aligned");
  const CocoWs w = coco_ws(workspace, p.n_det, p.n_gt, p.n_cats);
  CVB_REQUIRE(w.total > 0, "coco_eval_bbox: CUB could not size its temporary storage for %d detections", p.n_det);
  CVB_REQUIRE(ws_bytes >= w.total, "coco_eval_bbox: workspace of %zu bytes < %zu", ws_bytes, w.total);
  cudaStream_t st = as_stream(stream);
  const int n = p.n_det;
  CVB_CHECK_CUDA(cudaMemsetAsync(w.npig, 0, (size_t)p.n_cats * kCocoA * 4, st));
  if (n > 0) {
    CVB_CHECK_CUDA(cudaMemsetAsync(det_masks, 0, (size_t)n * kCocoA * 4, st));
    if (p.n_gt > 0) CVB_CHECK_CUDA(cudaMemsetAsync(w.gt_matched, 0, (size_t)p.n_gt * kScans, st));
    const int blocks = ceil_div(n, 256);
    coco_keys_kernel<<<blocks, 256, 0, st>>>(n, p.n_images, det_img, det_cat, det_score, w.keys_in, w.vals_in);
    size_t tb = w.cub_bytes;
    CVB_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(w.cub_tmp, tb, w.keys_in, w.keys, w.vals_in, w.order, n, 0, 64, st));
    coco_heads_kernel<<<blocks, 256, 0, st>>>(n, w.keys, w.flags, w.vals_in);
    tb = w.cub_bytes;
    CVB_CHECK_CUDA(cub::DeviceSelect::Flagged(w.cub_tmp, tb, w.vals_in, w.flags, w.seg_start, w.num_segs, n, st));
    coco_match_kernel<<<min(n, kSmCount * 8), kMatchThreads, 0, st>>>(p, w.keys, w.order, w.seg_start, w.num_segs, gt_key, gt_box, gt_area,
                                                                       gt_crowd, det_box, w.gt_matched, w.key2_in, w.det_rank, det_masks);
    tb = w.cub_bytes;
    CVB_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(w.cub_tmp, tb, w.key2_in, w.key2, w.order, w.order2, n, 0, 64, st));
    count_launch(3);
  }
  if (p.n_gt > 0) {
    coco_npig_kernel<<<ceil_div(p.n_gt, 256), 256, 0, st>>>(p, gt_key, gt_area, gt_crowd, img_evaluated, w.npig);
    count_launch();
  }
  coco_accumulate_kernel<<<p.n_cats * kCocoA * kCocoM, kAccThreads, 0, st>>>(p, w.key2, w.order2, w.det_rank, det_masks, w.npig, precision,
                                                                            recall);
  coco_summarize_kernel<<<12, kSumThreads, 0, st>>>(p.n_cats, precision, recall, stats);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch(2);
  return CVB_OK;
}
