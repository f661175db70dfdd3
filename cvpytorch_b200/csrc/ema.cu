// Model EMA update (src/utils/ema.py ModelEMA.update): every floating state_dict entry of one EMA step in ONE launch.
//
// The reference runs, per entry, `item *= decay; item += (1 - decay) * src` as three fp32 ATen ops with the Python scalars rounded to
// float: e = fl(e * d), then e = fl(e + fl(m * c)) with d = (float)decay and c = (float)(1.0 - decay) (the difference taken in double on
// the host).  ema_step below is that sequence with explicitly rounded operations, so nothing contracts into an FMA and the result is
// bitwise the reference's on the same GPU.
//
// Work layout: the table holds one EmaRecord per entry; entry i is cut into chunks of kEmaChunk elements numbered from first_chunk.  A
// fixed grid walks the (entry, chunk) work items grid-stride and finds each item's entry by a binary search over first_chunk (the table is
// a few KB and stays in L1 / L2).  A chunk whose ema and src pointers are both 16-byte aligned moves float4s, kEmaVec loads of each tensor
// in flight per thread; any other chunk, and the last numel % 4 elements of an entry, go element by element.  No atomics, no host sync.
#include <vector>

#include "internal.h"

namespace cvb {

constexpr int kEmaThreads = 256;
constexpr int kEmaVec = 4;                                    // float4 per thread per chunk
constexpr int64_t kEmaChunk = (int64_t)kEmaThreads * 4 * kEmaVec;  // 4096 elements
constexpr int kEmaGrid = kSmCount * 4;

struct EmaRecord {
  float* ema;
  const float* src;
  int64_t numel;
  int64_t first_chunk;  // work items of the entries before this one
};
static_assert(sizeof(EmaRecord) == CVB_EMA_TABLE_ENTRY_BYTES, "the device table format is part of the C ABI's size contract");

__device__ __forceinline__ float ema_step(float e, float m, float d, float c) { return __fadd_rn(__fmul_rn(e, d), __fmul_rn(m, c)); }

__global__ void __launch_bounds__(kEmaThreads) ema_update_kernel(const EmaRecord* __restrict__ table, int n, float d, float c) {
  const int64_t total = table[n - 1].first_chunk + (table[n - 1].numel + kEmaChunk - 1) / kEmaChunk;
  for (int64_t w = blockIdx.x; w < total; w += gridDim.x) {
    const EmaRecord r = owning_record(table, n, w);
    const int64_t begin = (w - r.first_chunk) * kEmaChunk;
    const int len = (int)min(kEmaChunk, r.numel - begin);
    float* e = r.ema + begin;
    const float* s = r.src + begin;
    int scalar_from = 0;
    if (is_aligned(e, 16) & is_aligned(s, 16)) {  // (& rather than &&: one branch-free test)
      float4* e4 = reinterpret_cast<float4*>(e);
      const float4* s4 = reinterpret_cast<const float4*>(s);
      const int nvec = len >> 2;
      float4 ev[kEmaVec], sv[kEmaVec];
#pragma unroll
      for (int k = 0; k < kEmaVec; ++k) {
        const int i = threadIdx.x + k * kEmaThreads;
        if (i < nvec) {
          ev[k] = e4[i];
          sv[k] = s4[i];
        }
      }
#pragma unroll
      for (int k = 0; k < kEmaVec; ++k) {
        const int i = threadIdx.x + k * kEmaThreads;
        if (i < nvec)
          e4[i] = make_float4(ema_step(ev[k].x, sv[k].x, d, c), ema_step(ev[k].y, sv[k].y, d, c), ema_step(ev[k].z, sv[k].z, d, c),
                              ema_step(ev[k].w, sv[k].w, d, c));
      }
      scalar_from = nvec << 2;
    }
    for (int i = scalar_from + threadIdx.x; i < len; i += kEmaThreads) e[i] = ema_step(e[i], s[i], d, c);
  }
}

}  // namespace cvb

using namespace cvb;

extern "C" int cvb_ema_table_upload(const CvbEmaEntry* entries, int32_t n, void* table, void* stream) {
  CVB_REQUIRE(entries && table, "ema_table_upload: null pointer");
  CVB_REQUIRE(n > 0, "ema_table_upload: n_entries must be > 0 (n=%d)", n);
  CVB_REQUIRE(is_aligned(table, 16), "ema_table_upload: table must be 16-byte aligned");
  std::vector<EmaRecord> recs(n);
  int64_t chunks = 0;
  for (int i = 0; i < n; ++i) {
    const CvbEmaEntry& x = entries[i];
    CVB_REQUIRE(x.numel >= 0, "ema_table_upload: entry %d has numel %lld < 0", i, (long long)x.numel);
    CVB_REQUIRE(x.numel == 0 || (x.ema && x.src), "ema_table_upload: entry %d has a null pointer", i);
    recs[i] = EmaRecord{x.ema, x.src, x.numel, chunks};
    chunks += (x.numel + kEmaChunk - 1) / kEmaChunk;
  }
  // (pageable source: the copy is staged before cudaMemcpyAsync returns, so recs may go out of scope)
  CVB_CHECK_CUDA(cudaMemcpyAsync(table, recs.data(), (size_t)n * sizeof(EmaRecord), cudaMemcpyHostToDevice, as_stream(stream)));
  return CVB_OK;
}

extern "C" int cvb_ema_update(const void* table, int32_t n, float decay, float one_minus_decay, void* stream) {
  CVB_REQUIRE(table, "ema_update: null pointer");
  CVB_REQUIRE(n > 0, "ema_update: n_entries must be > 0 (n=%d)", n);
  CVB_REQUIRE(is_aligned(table, 16), "ema_update: table must be 16-byte aligned");
  ema_update_kernel<<<kEmaGrid, kEmaThreads, 0, as_stream(stream)>>>(static_cast<const EmaRecord*>(table), n, decay, one_minus_decay);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}
