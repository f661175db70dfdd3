// Internal helpers shared by the translation units of libcvb200.so (not part of the C ABI).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#ifdef __CUDACC__
#include <cuda_fp16.h>
#endif

#include "../../include/cvb200.h"

namespace cvb {

// SM count of the H100 SXM: caps the grids of the grid-stride element-wise kernels (a few CTAs per SM)
constexpr int kSmCount = 132;

// thread-local error text returned by cvb_last_error_string()
int set_error(int code, const char* fmt, ...);
void count_launch(int n = 1);

#define CVB_CHECK_CUDA(expr)                                                                       \
  do {                                                                                             \
    cudaError_t _e = (expr);                                                                       \
    if (_e != cudaSuccess)                                                                         \
      return ::cvb::set_error(CVB_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

#define CVB_REQUIRE(cond, ...)                                       \
  do {                                                               \
    if (!(cond)) return ::cvb::set_error(CVB_ERR_INVALID, __VA_ARGS__); \
  } while (0)

// Tiled tensor map with unit element strides, no interleave, 256-byte L2 promotion and zero OOB fill: strides_bytes has rank - 1 entries.
// A missing driver entry point is CVB_ERR_NO_DEVICE, a refused encoding CVB_ERR_CUDA with the extents and box in the message.
int encode_map(CUtensorMap* m, CUtensorMapDataType dt, int rank, const void* base, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
               const cuuint32_t* box, CUtensorMapSwizzle swz);

// SM count of the current device, queried once per process; 0 (with CVB_ERR_NO_DEVICE set) when there is no device.
int sm_count();

// Opt-in of kernel fn to `bytes` of dynamic shared memory per CTA (above the default 48 KB).
template <typename F>
inline cudaError_t opt_in_smem(F* fn, int bytes) {
  return cudaFuncSetAttribute(reinterpret_cast<const void*>(fn), cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
}

inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// p is a multiple of a (a power of two)
__host__ __device__ inline bool is_aligned(const void* p, size_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }

// Lays the pieces of a workspace out one after another, each on a 256-byte boundary.  Constructed on nullptr it only sizes: take()
// returns nullptr and bytes() is what the workspace needs.
class WsCarver {
 public:
  explicit WsCarver(void* base) : base_(static_cast<char*>(base)) {}
  void* take(size_t bytes) {
    char* r = base_ ? base_ + off_ : nullptr;
    off_ = align_up(off_ + bytes, 256);
    return r;
  }
  size_t bytes() const { return off_; }

 private:
  char* base_;
  size_t off_ = 0;
};

// bytes per element of a CVB_SEG_* label dtype code
inline int seg_label_bytes(int32_t code) { return code == CVB_SEG_U8 ? 1 : code == CVB_SEG_I32 ? 4 : 8; }

// Division by a run-time constant d >= 1 with one multiply-high: magic = ceil(2^32 / d) is exact for 0 <= x < x_end while
// x_end * d < 2^32; otherwise magic = 0 selects real division, and magic = 1 means d == 1.
inline uint32_t fast_div_magic(int d, unsigned long long x_end) {
  if (d <= 1) return 1u;
  if (x_end * (unsigned long long)d >= 0xFFFFFFFFULL) return 0u;
  return (uint32_t)((0x100000000ULL + (unsigned long long)d - 1) / (unsigned long long)d);
}
#ifdef __CUDACC__
__device__ __forceinline__ int fast_div(int x, int d, uint32_t magic) { return magic == 1u ? x : (magic ? (int)__umulhi((uint32_t)x, magic) : x / d); }
#endif

// NMS score histogram (shared by nms.cu, the decode kernels and the fused-decode conv epilogue): kNmsBins bins per image
constexpr int kNmsBins = 16384;
#ifdef __CUDACC__
// Histogram bin of a score: its fp32 bits >> 17, monotone in non-negative scores; sign-bit patterns clamp to the last bin.
__device__ __forceinline__ uint32_t nms_score_bin(float score) { return min(__float_as_uint(score) >> 17, (uint32_t)(kNmsBins - 1)); }

// ++hist[nms_score_bin(sc)] of a shared-memory histogram iff `on`, as one predicated red.shared with no branch (a C++ `if (on)
// atomicAdd(...)` compiles to a ~14-instruction divergent region per score, which dominated the fused-decode epilogue).  The bin
// formula must match nms_score_bin above.
__device__ __forceinline__ void hist_inc_if(uint32_t hist_smem_addr, float sc, bool on) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t.reg .b32 t;\n\tsetp.ne.b32 p, %2, 0;\n\tshr.b32 t, %1, 17;\n\tmin.u32 t, t, %3;\n\tmad.lo.u32 t, t, 4, %0;\n\t"
      "@p red.shared.add.u32 [t], 1;\n\t}\n"
      ::"r"(hist_smem_addr), "r"(__float_as_uint(sc)), "r"((uint32_t)on), "n"(kNmsBins - 1)
      : "memory");
}

// The NMS score pre-pass: what a decode kernel or the NMS counting pass builds for every z row, and what cvb_yolo_nms then trusts
// (hist_ready = 1).  Each lane of the row's warp counts its scores into `best` (starting from 0) with nms_count_score, then
// nms_finish_row gives the row's rowmax entry.  multi: one histogram entry per score > conf; else one per row with a best score > conf.
__device__ __forceinline__ void nms_count_score(uint32_t* hist, float sc, float conf, bool multi, float& best) {
  if (multi && sc > conf) atomicAdd(&hist[nms_score_bin(sc)], 1u);
  best = fmaxf(best, sc);
}

// Warp-wide: the row's best score if it is > conf, else 0 (every lane gets it).
__device__ __forceinline__ float nms_finish_row(uint32_t* hist, float best, float conf, bool multi, int lane) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) best = fmaxf(best, __shfl_xor_sync(0xffffffffu, best, o));
  if (!(best > conf)) best = 0.0f;
  if (!multi && lane == 0 && best > conf) atomicAdd(&hist[nms_score_bin(best)], 1u);
  return best;
}

// A CTA's shared-memory histogram: zeroed before the CTA counts into it, and its non-empty bins added to the image's global
// histogram once at the end (keeps the hot bins out of global atomics).
template <int kThreads>
__device__ __forceinline__ void nms_hist_clear(uint32_t* s_hist) {
  for (int i = threadIdx.x; i < kNmsBins; i += kThreads) s_hist[i] = 0;
  __syncthreads();
}
template <int kThreads>
__device__ __forceinline__ void nms_hist_flush(const uint32_t* s_hist, uint32_t* g_hist) {
  __syncthreads();
  for (int i = threadIdx.x; i < kNmsBins; i += kThreads) {
    const uint32_t c = s_hist[i];
    if (c) atomicAdd(&g_hist[i], c);
  }
}
#endif
constexpr int kNmsCap = 65536;   // candidate key capacity per image (phase B)
constexpr int kNmsCapA = 4096;   // phase-A candidate capacity = one shared-memory sort chunk

// NMS workspace layout (bytes): [hist B*kNmsBins u32][6 slots of B u32][keysB B*kNmsCap u64][keysA B*kNmsCapA u64][rowmax B*A f32]
// rowmax[b][anchor] = best score (obj*cls, > conf) of the anchor row, 0 when it has no candidate: written by the pass that
// builds the histogram (decode kernel or the NMS count pass) and lets the emit passes skip rows below the threshold bin.
inline size_t nms_ws_head_bytes(int B) { return align_up((size_t)B * kNmsBins * 4, 256) + 6 * align_up((size_t)B * 4, 256); }
inline size_t nms_ws_rowmax_offset(int B) { return nms_ws_head_bytes(B) + (size_t)B * (kNmsCap + kNmsCapA) * 8; }
inline float* nms_ws_rowmax(void* ws, int B) { return ws ? reinterpret_cast<float*>(static_cast<uint8_t*>(ws) + nms_ws_rowmax_offset(B)) : nullptr; }

// A decode level writes the z rows [z_off, z_off + rows) of each image, which must lie inside the image's z_rows.
inline int check_level_rows(const char* op, long long z_off, long long rows, long long z_rows) {
  CVB_REQUIRE(z_off >= 0 && z_off + rows <= z_rows, "%s: level rows [%lld, %lld) outside z's %lld rows", op, z_off, z_off + rows, z_rows);
  return CVB_OK;
}

#ifdef __CUDACC__
// The one fp32 -> split16 (hi, lo) conversion, for a pair of values (one F2FP per plane).  hi = fp16_rn(x) and lo = fp16_rn(x - hi), both
// saturating to +-65504 (cvt .satfinite): |x| <= 65504 is kept to ~22 bits, up to 131008 survives with lo carrying the excess, larger values
// and +-inf saturate to +-131008, and NaN stays NaN (DESIGN.md 2).  Every kernel that stores split16 calls it.
__device__ __forceinline__ void split_pair(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(x1), "f"(x0));
  const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hi));
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(x1 - hf.y), "f"(x0 - hf.x));
}

// Max that propagates NaN like F.max_pool2d: once the running maximum m is NaN it stays NaN.
__device__ __forceinline__ float nan_max(float m, float v) { return (v > m || v != v) ? v : m; }

// sigmoid with two MUFU ops (ex2, rcp), |rel err| ~ 2^-22 (the reference's own CPU sigmoid is ~1 ulp; parity budget 1e-3).  Shared by
// the YOLOv5 / YOLOX / FCOS decode kernels so that every pass that recomputes a score gets the identical value.
__device__ __forceinline__ float sigmoid_fast(float x) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * -1.4426950408889634f));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
  return r;
}

// The YOLOv5 decode of one z row and its NMS score, written once for the stand-alone decode kernel, the fused-decode conv epilogue
// and the NMS passes that recompute scores from z, which must all produce the same fp32 bits.  Reference: y = x.sigmoid();
// xy = (y*2 - 0.5 + grid) * stride; wh = (y*2)**2 * anchor_grid (yolov5_detect.py:50-53); score = cls * obj (yolov5.py:106).
__device__ __forceinline__ float yolo_xy(float y, float grid, float stride) {
  return __fmul_rn(__fadd_rn(__fsub_rn(__fmul_rn(y, 2.0f), 0.5f), grid), stride);
}
__device__ __forceinline__ float yolo_wh(float y, float anchor) {
  const float t2 = __fmul_rn(y, 2.0f);
  return __fmul_rn(__fmul_rn(t2, t2), anchor);
}
__device__ __forceinline__ float yolo_score(float cls, float obj) { return __fmul_rn(cls, obj); }

// Source taps of output index dst of a bilinear resize with align_corners = False, PyTorch's upsample_bilinear2d with size= given:
// scale = (float)in / out, src = max((dst + 0.5) * scale - 0.5, 0), i0 = (int)src, i1 = i0 + (i0 < in - 1), l1 = src - i0 (the weight of
// i1; i0's is 1 - l1).  Shared by the split16 resize, the fused upsample + argmax and the segmentation loss, so that they interpolate alike.
__device__ __forceinline__ void bilinear_src(int dst, float scale, int in_size, int* i0, int* i1, float* l1) {
  float s = fmaxf(((float)dst + 0.5f) * scale - 0.5f, 0.0f);
  int a = (int)s;
  if (a > in_size - 1) a = in_size - 1;
  *i0 = a;
  *i1 = a + ((a < in_size - 1) ? 1 : 0);
  *l1 = s - (float)a;
}

// The training losses' fp32 sigmoid and BCEWithLogits (pos_weight 1), shared by yolox_loss.cu and yolov5_loss.cu:
// BCEWithLogits(x, t) = (1 - t) x + m + log(exp(-m) + exp(-x - m)), m = max(-x, 0)
__device__ __forceinline__ float sigmoidf(float x) { return 1.0f / (1.0f + expf(-x)); }
__device__ __forceinline__ float bce_logits(float x, float t) {
  const float m = fmaxf(-x, 0.0f);
  return (1.0f - t) * x + m + logf(expf(-m) + expf(-x - m));
}

// The one fp64 summation order of the losses' per-CTA and final reductions (DESIGN.md 2), so that every loss adds alike: a warp adds its
// lanes by an xor butterfly (offsets 16, 8, 4, 2, 1; every lane ends with the warp total), then the warp totals are added in ascending warp
// order starting from 0.0.
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Block-wide sum of N values per thread of a kThreads-thread CTA, in the order above; thread 0 gets the totals in v.  red is shared
// [kThreads / 32][N]; the leading barrier lets calls follow one another on the same red.  (Only thread 0 adds the warp totals: every
// thread doing so costs kThreads * N fp64 adds per CTA, which slowed the 4096-CTA segmentation forward by about 1 us.)
template <int kThreads, int N>
__device__ __forceinline__ void block_sum(double (&v)[N], double (*red)[N]) {
  __syncthreads();
#pragma unroll
  for (int k = 0; k < N; ++k) v[k] = warp_sum(v[k]);
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int k = 0; k < N; ++k) red[threadIdx.x >> 5][k] = v[k];
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
#pragma unroll
  for (int k = 0; k < N; ++k) {
    double t = 0.0;
    for (int w = 0; w < kThreads / 32; ++w) t += red[w][k];
    v[k] = t;
  }
}

// The record of a work table (ema.cu, sgd.cu) that owns work item w: the last of table[0, n) with first_chunk <= w, first_chunk being
// non-decreasing from 0 (an entry with no items shares its first_chunk with the next one, which wins).
template <typename R>
__device__ __forceinline__ R owning_record(const R* __restrict__ table, int n, int64_t w) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (table[mid].first_chunk <= w) lo = mid;
    else hi = mid - 1;
  }
  return table[lo];
}
#endif

}  // namespace cvb
