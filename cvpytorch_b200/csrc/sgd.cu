// SGD step (torch.optim.SGD under torch.amp.GradScaler, as src/optimizers/__init__.py build_optimizer sets it up): every parameter of
// every group in ONE launch, with GradScaler's unscale and overflow skip read from the device.
//
// Per element, in fp32 with the Python scalars rounded to float (the reference's GradScaler.unscale_, then _multi_tensor_sgd):
//   g1  = g * inv_scale                      inv_scale = (float)(1.0 / (double)*grad_scale), only with a grad_scale
//   d   = g1 + wd * p                        only if wd != 0
//   buf = buf * m + d  (first step: d)       only if m != 0; buf * m is rounded before the add (_foreach_mul_, then _foreach_add_)
//   d   = nesterov ? d + m * buf : buf       only if m != 0
//   p   = p + (-lr) * d
// ATen's foreach `a + alpha * b` (the weight decay, the Nesterov term and the parameter update) is one fused multiply-add on the H100:
// torch._foreach_add_ and Tensor.add_ with alpha matched fmaf on all of 2^20 random pairs and missed the separately rounded form on 300,241
// of them.  So add_scaled below is __fmaf_rn, and every other product and sum is rounded on its own (__fmul_rn / __fadd_rn, --fmad=false).
// The result is bitwise the reference's on the same GPU.  A non-zero *found_inf makes the whole launch a no-op, as GradScaler skips optimizer.step().
//
// Work layout as ema.cu: one SgdRecord per parameter, cut into kSgdChunk-element chunks numbered from first_chunk (an empty parameter
// still owns one chunk, so its buffer becomes valid as the reference's clone of an empty gradient does).  A fixed grid walks the
// (entry, chunk) items grid-stride and binary-searches first_chunk.  float4 where param, grad and buffer are all 16-byte aligned, element by
// element otherwise.  The group hyper-parameters arrive by value in a __grid_constant__ argument, so a new lr costs no copy.
//
// Momentum buffer validity lives on the device, one int32 flag per chunk: 0 until the first step that was not skipped has written that
// chunk's buffer (the reference clones d into a new buffer there), 1 after.  Each chunk is read and written by one CTA, so the flag needs no
// ordering between CTAs: its threads read it, and thread 0 sets it after a barrier.  No atomics, no host sync, CUDA-graph capturable.
#include <vector>

#include "internal.h"

namespace cvb {

constexpr int kSgdThreads = 256;
constexpr int kSgdVec = 4;                                        // float4 per thread per chunk
constexpr int64_t kSgdChunk = (int64_t)kSgdThreads * 4 * kSgdVec;  // 4096 elements
static_assert(kSgdChunk == CVB_SGD_CHUNK, "the flag count per parameter is part of the C ABI");
constexpr int kSgdGrid = kSmCount * 4;

struct SgdRecord {
  float* param;
  const float* grad;
  float* buf;
  int32_t* valid;
  int64_t numel;
  int64_t first_chunk;  // work items of the entries before this one
  int32_t group;
  int32_t pad_[3];
};
static_assert(sizeof(SgdRecord) == CVB_SGD_TABLE_ENTRY_BYTES, "the device table format is part of the C ABI's size contract");

// the groups by value: 256 groups (4 KB) cover the reference's models; larger optimisers take the 16 KB form
template <int kCap>
struct SgdGroups {
  CvbSgdGroup g[kCap];
};
static_assert(sizeof(SgdGroups<CVB_SGD_MAX_GROUPS>) <= 32764 - 64, "kernel arguments must fit CUDA 12.1+'s 32 KB limit");

__device__ __forceinline__ int64_t sgd_items(int64_t numel) { return numel > kSgdChunk ? (numel + kSgdChunk - 1) / kSgdChunk : 1; }

// a + alpha * b as ATen's foreach add with alpha computes it: one fused multiply-add
__device__ __forceinline__ float add_scaled(float a, float alpha, float b) { return __fmaf_rn(alpha, b, a); }

struct SgdConsts {
  float lr_neg, wd, m, inv;
  bool scaled, decay, momentum, nesterov, have_buf;
};

__device__ __forceinline__ void sgd_element(float& p, float g, float& b, const SgdConsts& k) {
  float d = k.scaled ? __fmul_rn(g, k.inv) : g;
  if (k.decay) d = add_scaled(d, k.wd, p);
  if (k.momentum) {
    b = k.have_buf ? __fadd_rn(__fmul_rn(b, k.m), d) : d;
    d = k.nesterov ? add_scaled(d, k.m, b) : b;
  }
  p = add_scaled(p, k.lr_neg, d);
}

template <int kCap>
__global__ void __launch_bounds__(kSgdThreads, 4)  // 64 registers, no spills: the grid's 4 CTAs per SM are resident
    sgd_step_kernel(const SgdRecord* __restrict__ table, int n, const __grid_constant__ SgdGroups<kCap> groups,
                    const float* __restrict__ grad_scale, const float* __restrict__ found_inf) {
  if (found_inf && *found_inf != 0.f) return;
  SgdConsts k;
  k.scaled = grad_scale != nullptr;
  k.inv = k.scaled ? __double2float_rn(1.0 / (double)*grad_scale) : 1.f;
  const int64_t total = table[n - 1].first_chunk + sgd_items(table[n - 1].numel);
  for (int64_t w = blockIdx.x; w < total; w += gridDim.x) {
    const SgdRecord r = owning_record(table, n, w);
    const CvbSgdGroup h = groups.g[r.group];
    k.lr_neg = -h.lr;
    k.wd = h.weight_decay;
    k.m = h.momentum;
    k.decay = (h.flags & CVB_SGD_WEIGHT_DECAY) != 0;
    k.momentum = (h.flags & CVB_SGD_MOMENTUM) != 0;
    k.nesterov = (h.flags & CVB_SGD_NESTEROV) != 0;
    const int64_t chunk = w - r.first_chunk;
    const int64_t begin = chunk * kSgdChunk;
    const int len = (int)max((int64_t)0, min(kSgdChunk, r.numel - begin));
    k.have_buf = k.momentum && r.valid[chunk] != 0;
    float* p = r.param + begin;
    const float* g = r.grad + begin;
    float* b = k.momentum ? r.buf + begin : nullptr;
    int scalar_from = 0;
    if (is_aligned(p, 16) & is_aligned(g, 16) & is_aligned(b, 16)) {  // (& rather than &&: one branch-free test)
      float4* p4 = reinterpret_cast<float4*>(p);
      const float4* g4 = reinterpret_cast<const float4*>(g);
      float4* b4 = reinterpret_cast<float4*>(b);
      const int nvec = len >> 2;
      float4 pv[kSgdVec], gv[kSgdVec], bv[kSgdVec];
#pragma unroll
      for (int v = 0; v < kSgdVec; ++v) {
        const int i = threadIdx.x + v * kSgdThreads;
        if (i < nvec) {
          pv[v] = p4[i];
          gv[v] = g4[i];
          bv[v] = k.have_buf ? b4[i] : make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
#pragma unroll
      for (int v = 0; v < kSgdVec; ++v) {
        const int i = threadIdx.x + v * kSgdThreads;
        if (i < nvec) {
          sgd_element(pv[v].x, gv[v].x, bv[v].x, k);
          sgd_element(pv[v].y, gv[v].y, bv[v].y, k);
          sgd_element(pv[v].z, gv[v].z, bv[v].z, k);
          sgd_element(pv[v].w, gv[v].w, bv[v].w, k);
          p4[i] = pv[v];
          if (k.momentum) b4[i] = bv[v];
        }
      }
      scalar_from = nvec << 2;
    }
    for (int i = scalar_from + threadIdx.x; i < len; i += kSgdThreads) {
      float pe = p[i], be = k.have_buf ? b[i] : 0.f;
      sgd_element(pe, g[i], be, k);
      p[i] = pe;
      if (k.momentum) b[i] = be;
    }
    if (k.momentum) {  // uniform across the CTA: every thread has read the flag before thread 0 sets it
      __syncthreads();
      if (threadIdx.x == 0 && !k.have_buf) r.valid[chunk] = 1;
    }
  }
}

template <int kCap>
int launch_sgd(const void* table, int32_t n, const CvbSgdGroup* groups, int32_t n_groups, const float* grad_scale, const float* found_inf,
               void* stream) {
  SgdGroups<kCap> g{};
  for (int i = 0; i < n_groups; ++i) g.g[i] = groups[i];
  sgd_step_kernel<kCap><<<kSgdGrid, kSgdThreads, 0, as_stream(stream)>>>(static_cast<const SgdRecord*>(table), n, g, grad_scale, found_inf);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}

}  // namespace cvb

using namespace cvb;

extern "C" int cvb_sgd_table_upload(const CvbSgdEntry* entries, int32_t n, int32_t n_groups, void* table, void* stream) {
  CVB_REQUIRE(entries && table, "sgd_table_upload: null pointer");
  CVB_REQUIRE(n > 0, "sgd_table_upload: n_entries must be > 0 (n=%d)", n);
  CVB_REQUIRE(n_groups > 0 && n_groups <= CVB_SGD_MAX_GROUPS, "sgd_table_upload: n_groups must be in [1, %d] (n_groups=%d)", CVB_SGD_MAX_GROUPS,
              n_groups);
  CVB_REQUIRE(is_aligned(table, 16), "sgd_table_upload: table must be 16-byte aligned");
  std::vector<SgdRecord> recs(n);
  int64_t chunks = 0;
  for (int i = 0; i < n; ++i) {
    const CvbSgdEntry& x = entries[i];
    CVB_REQUIRE(x.numel >= 0, "sgd_table_upload: entry %d has numel %lld < 0", i, (long long)x.numel);
    CVB_REQUIRE(x.group >= 0 && x.group < n_groups, "sgd_table_upload: entry %d has group %d outside [0, %d)", i, x.group, n_groups);
    CVB_REQUIRE(x.numel == 0 || (x.param && x.grad), "sgd_table_upload: entry %d has a null pointer", i);
    CVB_REQUIRE(!x.momentum_buffer || x.valid, "sgd_table_upload: entry %d has a momentum buffer without valid flags", i);
    CVB_REQUIRE(!x.valid || x.numel == 0 || x.momentum_buffer, "sgd_table_upload: entry %d has valid flags without a momentum buffer", i);
    recs[i] = SgdRecord{x.param, x.grad, x.momentum_buffer, x.valid, x.numel, chunks, x.group, {0, 0, 0}};
    chunks += x.numel > kSgdChunk ? (x.numel + kSgdChunk - 1) / kSgdChunk : 1;
  }
  // (pageable source: the copy is staged before cudaMemcpyAsync returns, so recs may go out of scope)
  CVB_CHECK_CUDA(cudaMemcpyAsync(table, recs.data(), (size_t)n * sizeof(SgdRecord), cudaMemcpyHostToDevice, as_stream(stream)));
  return CVB_OK;
}

extern "C" int cvb_sgd_step(const void* table, int32_t n, const CvbSgdGroup* groups, int32_t n_groups, const float* grad_scale,
                            const float* found_inf, void* stream) {
  CVB_REQUIRE(table && groups, "sgd_step: null pointer");
  CVB_REQUIRE(n > 0, "sgd_step: n_entries must be > 0 (n=%d)", n);
  CVB_REQUIRE(n_groups > 0 && n_groups <= CVB_SGD_MAX_GROUPS, "sgd_step: n_groups must be in [1, %d] (n_groups=%d)", CVB_SGD_MAX_GROUPS, n_groups);
  CVB_REQUIRE(is_aligned(table, 16), "sgd_step: table must be 16-byte aligned");
  if (n_groups <= 256) return launch_sgd<256>(table, n, groups, n_groups, grad_scale, found_inf, stream);
  return launch_sgd<CVB_SGD_MAX_GROUPS>(table, n, groups, n_groups, grad_scale, found_inf, stream);
}
