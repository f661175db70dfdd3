// Segmentation confusion matrix (src/evaluator/eval_segmentation.py SegmentationEvaluator._generate_matrix + update): one stream-ordered
// pass over a pair of label maps that adds their pixel counts to a uint64 [nc, nc] matrix on the device, with no host sync.
//
// The reference's rule, for every pixel with 0 <= gt < nc: flat = nc * gt + pred in int64 (numpy's wrap-around included), and
// bincount(flat, minlength=nc²).reshape(nc, nc).  A flat index in [0, nc²) counts in that bin, so an out-of-range prediction aliases
// into a neighbouring row as it does in numpy; a flat index < 0 (bincount raises) sets bit 0 of *err, one >= nc² (reshape raises) bit 1.
//
// Work layout: a grid-stride pass over "steps" of E = 16 / max(sizeof gt, sizeof pred) pixels.  The wider map moves in 16-byte vectors
// and the narrower one in the matching E-element vector, so every load instruction of a warp covers one contiguous span of each map.
// The vector path starts at the first pixel where both maps are aligned to their vector width (the host finds it); the pixels before it
// and after the last whole step, or every pixel when the two maps can never be aligned together, are read one by one.  Each CTA counts
// into uint32 bins in shared memory: R replicas of the nc² bins (R up to 32 for small nc, lane l uses replica l % R), with an odd
// replica stride so that the lanes of a warp counting one dominant class hit R different banks.  The CTA then sums its replicas and
// flushes each non-zero bin with one 64-bit atomicAdd; integer adds commute, so the matrix is exact and the same on every run.  A CTA
// counts at most n <= 2^31 - 1 pixels, so no uint32 bin can overflow.
#include "internal.h"

namespace cvb {

constexpr int kSegThreads = 256;
// steps in flight per thread: 64 bytes of the wider map, or 2 x 16 pixels of two uint8 maps (four would spill under 4 CTAs per SM)
template <int E>
constexpr int kSegUnroll = E >= 16 ? 2 : 4;
constexpr int kSegMaxReplicas = 32;            // one per lane
constexpr int kSegReplicaBytes = 48 * 1024;    // shared memory given to replicas, so that four CTAs fit on an SM
constexpr int kSegSmemOptinBytes = 232448;     // the sm_90 opt-in shared memory per CTA (227 KB)

constexpr int seg_isqrt(int x, int r = 0) { return (r + 1) * (r + 1) > x ? r : seg_isqrt(x, r + 1); }
// the largest nc whose nc² uint32 bins fit one CTA's shared memory (241 on sm_90): larger nc are refused, there is no global fallback
constexpr int kSegNcMax = seg_isqrt(kSegSmemOptinBytes / 4);
static_assert(kSegNcMax * kSegNcMax * 4 <= kSegSmemOptinBytes && (kSegNcMax + 1) * (kSegNcMax + 1) * 4 > kSegSmemOptinBytes, "NC_MAX");
static_assert(kSegNcMax >= 182, "ADE20K (150) and COCO-Stuff (182) must fit");

template <typename T, int E>
struct alignas(sizeof(T) * E) SegPack {
  T v[E];
};

template <typename G, typename P>
__device__ __forceinline__ void seg_count(G g, P p, long long nc, long long nc2, uint32_t* hist, uint32_t& err) {
  const long long gi = (long long)g;
  if (gi >= 0 && gi < nc) {
    // int64 arithmetic that wraps like numpy's
    const long long flat = (long long)((unsigned long long)(nc * gi) + (unsigned long long)(long long)p);
    if ((unsigned long long)flat < (unsigned long long)nc2) atomicAdd(&hist[flat], 1u);
    else err |= flat < 0 ? 1u : 2u;
  }
}

template <typename G, typename P>
__global__ void __launch_bounds__(kSegThreads, 4) seg_confusion_kernel(const G* __restrict__ gt, const P* __restrict__ pred, long long n,
                                                                    long long head, long long steps, int nc, int replicas, int stride,
                                                                    unsigned long long* __restrict__ matrix, int* __restrict__ err_out) {
  constexpr int kW = sizeof(G) > sizeof(P) ? (int)sizeof(G) : (int)sizeof(P);
  constexpr int E = 16 / kW;
  constexpr int U = kSegUnroll<E>;
  extern __shared__ uint32_t s_hist[];
  const int nc2 = nc * nc;
  for (int i = threadIdx.x; i < replicas * stride; i += kSegThreads) s_hist[i] = 0;
  __syncthreads();
  uint32_t* hist = s_hist + (threadIdx.x & 31) % replicas * stride;
  uint32_t err = 0;

  const SegPack<G, E>* gv = reinterpret_cast<const SegPack<G, E>*>(gt + head);
  const SegPack<P, E>* pv = reinterpret_cast<const SegPack<P, E>*>(pred + head);
  const long long tile = (long long)gridDim.x * kSegThreads * U;
  for (long long s0 = (long long)blockIdx.x * kSegThreads * U + threadIdx.x; s0 < steps; s0 += tile) {
    SegPack<G, E> g[U];
    SegPack<P, E> p[U];
#pragma unroll
    for (int k = 0; k < U; ++k) {
      const long long s = s0 + (long long)k * kSegThreads;
      if (s < steps) {
        g[k] = gv[s];
        p[k] = pv[s];
      }
    }
#pragma unroll
    for (int k = 0; k < U; ++k) {
      if (s0 + (long long)k * kSegThreads < steps) {
#pragma unroll
        for (int j = 0; j < E; ++j) seg_count(g[k].v[j], p[k].v[j], nc, nc2, hist, err);
      }
    }
  }
  // the pixels outside the vector path: [0, head) and [head + steps * E, n)
  const long long tail = head + steps * E;
  const long long loose = head + (n - tail);
  for (long long j = (long long)blockIdx.x * kSegThreads + threadIdx.x; j < loose; j += (long long)gridDim.x * kSegThreads) {
    const long long i = j < head ? j : tail + (j - head);
    seg_count(gt[i], pred[i], nc, nc2, hist, err);
  }

  err = __reduce_or_sync(0xffffffffu, err);
  if (err && (threadIdx.x & 31) == 0) atomicOr(err_out, (int)err);
  __syncthreads();
  for (int b = threadIdx.x; b < nc2; b += kSegThreads) {
    uint32_t c = 0;
    for (int r = 0; r < replicas; ++r) c += s_hist[r * stride + b];
    if (c) atomicAdd(&matrix[b], (unsigned long long)c);
  }
}

template <typename G, typename P>
static int seg_launch(const void* gt, const void* pred, long long n, int nc, unsigned long long* matrix, int* err, cudaStream_t stream) {
  constexpr int kW = sizeof(G) > sizeof(P) ? (int)sizeof(G) : (int)sizeof(P);
  constexpr int E = 16 / kW;
  // first pixel where gt and pred both sit on their vector width (the step advances both by a whole vector); none: all scalar
  long long head = n;
  for (int h = 0; h < E; ++h) {
    if (is_aligned(static_cast<const G*>(gt) + h, E * sizeof(G)) && is_aligned(static_cast<const P*>(pred) + h, E * sizeof(P))) {
      head = h < n ? h : n;
      break;
    }
  }
  const long long steps = (n - head) / E;
  const int nc2 = nc * nc;
  const int stride = nc2 | 1;
  int replicas = kSegReplicaBytes / (stride * 4);
  replicas = replicas < 1 ? 1 : replicas > kSegMaxReplicas ? kSegMaxReplicas : replicas;
  const int smem = replicas * stride * 4;
  auto fn = seg_confusion_kernel<G, P>;
  CVB_CHECK_CUDA(opt_in_smem(fn, smem));
  const int sms = sm_count();
  if (sms == 0) return CVB_ERR_NO_DEVICE;
  int per_sm = 0;
  CVB_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, kSegThreads, smem));
  CVB_REQUIRE(per_sm > 0, "seg_confusion_update: %d bytes of shared memory do not fit a CTA", smem);
  constexpr int U = kSegUnroll<E>;
  const long long work = steps + (n - steps * E);  // vector steps + loose pixels
  long long grid = (work + (long long)kSegThreads * U - 1) / ((long long)kSegThreads * U);
  if (grid > (long long)sms * per_sm) grid = (long long)sms * per_sm;
  if (grid < 1) grid = 1;
  fn<<<(int)grid, kSegThreads, smem, stream>>>(static_cast<const G*>(gt), static_cast<const P*>(pred), n, head, steps, nc, replicas, stride,
                                              matrix, err);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}

template <typename G>
static int seg_dispatch_pred(const void* gt, const void* pred, int32_t pred_dtype, long long n, int nc, unsigned long long* matrix, int* err,
                             cudaStream_t stream) {
  switch (pred_dtype) {
    case CVB_SEG_U8: return seg_launch<G, uint8_t>(gt, pred, n, nc, matrix, err, stream);
    case CVB_SEG_I32: return seg_launch<G, int32_t>(gt, pred, n, nc, matrix, err, stream);
    default: return seg_launch<G, long long>(gt, pred, n, nc, matrix, err, stream);
  }
}

}  // namespace cvb

using namespace cvb;

extern "C" int32_t cvb_seg_confusion_nc_max(void) { return kSegNcMax; }

extern "C" int cvb_seg_confusion_update(const void* gt, int32_t gt_dtype, const void* pred, int32_t pred_dtype, int64_t n, int32_t nc,
                                        uint64_t* matrix, int32_t* err, void* stream) {
  CVB_REQUIRE(nc >= 1 && nc <= kSegNcMax, "seg_confusion_update: nc must be in [1, %d] (got %d)", kSegNcMax, nc);
  CVB_REQUIRE(n >= 0 && n <= 0x7fffffffLL, "seg_confusion_update: n must be in [0, 2^31 - 1] (got %lld)", (long long)n);
  const auto known = [](int32_t c) { return c == CVB_SEG_U8 || c == CVB_SEG_I32 || c == CVB_SEG_I64; };
  CVB_REQUIRE(known(gt_dtype) && known(pred_dtype), "seg_confusion_update: unknown dtype code (gt %d, pred %d)", gt_dtype, pred_dtype);
  if (n == 0) return CVB_OK;
  CVB_REQUIRE(gt && pred && matrix && err, "seg_confusion_update: null pointer");
  CVB_REQUIRE(is_aligned(gt, seg_label_bytes(gt_dtype)) && is_aligned(pred, seg_label_bytes(pred_dtype)),
              "seg_confusion_update: gt / pred not aligned to their element size");
  CVB_REQUIRE(is_aligned(matrix, 8) && is_aligned(err, 4),
              "seg_confusion_update: matrix must be 8-byte and err 4-byte aligned");
  unsigned long long* m = reinterpret_cast<unsigned long long*>(matrix);
  int* e = reinterpret_cast<int*>(err);
  const cudaStream_t s = as_stream(stream);
  switch (gt_dtype) {
    case CVB_SEG_U8: return seg_dispatch_pred<uint8_t>(gt, pred, pred_dtype, n, nc, m, e, s);
    case CVB_SEG_I32: return seg_dispatch_pred<int32_t>(gt, pred, pred_dtype, n, nc, m, e, s);
    default: return seg_dispatch_pred<long long>(gt, pred, pred_dtype, n, nc, m, e, s);
  }
}
