// Training-step kernels for the whole YOLOX network, backbone, neck and head (SURVEY.md 8 f-3): conv forward / backward-data /
// backward-weight as bf16 implicit GEMMs on wgmma + TMA, the BatchNorm(batch statistics) + SiLU forward / backward element-wise passes
// around them, and the Focus space-to-depth, SPPF pooling, neck upsample-concat and head prediction-conv passes.
//
// Replaces, for one  BaseConv = nn.Conv2d -> nn.BatchNorm2d -> SiLU  in training mode (src/models/modules/yolox_modules.py:35-55) and
// its autograd backward (what trainer.py:177-207 runs through cuDNN / ATen):
//   forward   y = conv(x, W)                         tconv_kernel            (M = 128 pixels, N = cout tile, K = taps x cin)
//             batch mean / var of y                  bn_stats_kernel + bn_finalize_kernel
//             a = silu(gamma * (y - mean) * rstd + beta)     bn_act_fwd_kernel<kActSilu>
//   backward  dz = da * silu'(z);  sum(dz), sum(dz * xhat)   bn_act_bwd_reduce_kernel   (or dz straight from the consumer's dgrad epilogue)
//             dy = gamma * rstd * (dz - mean(dz) - xhat * mean(dz * xhat))   bn_act_bwd_apply_kernel
//             dx = conv(dy, W rotated by 180 degrees, in/out swapped)   tconv_kernel again (optionally with the PRODUCER's SiLU' in the epilogue)
//             dW[co][tap][ci] = sum_pixels dy[p][co] * x[p + tap][ci]    twgrad_kernel   (K = pixels: both operands MN-major in shared memory)
// nn.SyncBatchNorm (statistics over every rank's pixels): bn_stats_kernel + bn_partial_kernel -> all-gather of the fp64 records ->
// bn_merge_kernel; backward bn_act_bwd_reduce_kernel -> all-reduce of the two sums -> bn_act_bwd_apply_kernel with the global count.
// YOLOv6 adds the same passes with ReLU (<kActRelu>), the RepVGG branch sum relu(bn3(y3) + bn1(y1) [+ bnid(x)]) with its backward
// (repvgg_*_kernel) and the ConvTranspose2d(c, c, 2, stride 2) scatter / gather around a 1x1 GEMM of 4c columns (convt_*_kernel).
// Synced, a RepVGG block takes one record per branch (the identity branch's on the block input) and one all-reduce of its [4][C] sums.
//
// Layout: activations and gradients are NHWC bf16, dense (pitch == C; C = 16, 32 or a multiple of 64, and TMA zero-fills a box's channels
// past a 16- or 32-channel C); weights bf16 [cout][kh*kw][kpad(cin)] (K-major rows, zero-padded to 64 channels), fp32 master weights / fp32
// weight gradients outside.  One TMA box {64 channels, TW, TH, NB} with TW*TH*NB == 128 pixels is at the same
// time a K-major A tile of the forward GEMM (row = pixel, 128 bytes of channels) and an MN-major operand of the weight-gradient GEMM
// (K = pixel rows); out-of-bounds pixels are zero-filled by TMA = the convolution padding, and contribute nothing to dW.
#include <cuda_bf16.h>

#include <cstring>
#include <new>

#include "internal.h"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace cvb {

constexpr int kTMmaWarps = 8;                 // warps 0..7: two MMA / epilogue warpgroups (accumulator rows 0-63 / 64-127)
constexpr int kTProducerWarp = kTMmaWarps;    // warp 8: TMA producer
constexpr int kTThreads = 32 * (kTMmaWarps + 1);
constexpr int kTStagesFwd = 4;
constexpr int kTStagesWg = 3;

// MN-major operand, 128-byte swizzle: rows are K indices (128 bytes = 64 MN elements each), 8-row groups SBO apart, the next 64 MN
// elements (panel) LBO apart  (canonical layout ((8,n),(8,k)):((1,LBO),(8,SBO)) in 16-byte units)
__device__ __forceinline__ uint64_t make_mnmajor_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
  d |= (uint64_t)(lbo_bytes >> 4) << 16;
  d |= (uint64_t)(sbo_bytes >> 4) << 32;
  d |= (uint64_t)2 << 61;
  return d;
}
__device__ __forceinline__ void tma_load_4d(const CUtensorMap* m, uint64_t* bar, void* smem, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
               ::"r"(smem_u32(smem)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* m, uint64_t* bar, void* smem, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
               ::"r"(smem_u32(smem)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
               : "memory");
}

struct alignas(64) TConvArgs {
  CUtensorMap tmA[4];  // activations {C, W, H, B}, box {64, TW, TH, NB}; stride 2: one map per (row parity, column parity) of the input
  CUtensorMap tmB;     // weights {K = taps * cin, cout}, box {64, BN}
  int tiles_w, tiles_h, tiles_b;
  int TW, TH, NB, H, W, B;   // H, W: the tile grid (output pixels of this launch)
  int cin, cout, taps;
  // tap t reads input map tap_map[t] at (w + tap_dw[t], h + tap_dh[t]) and the weight K block tap_wblk[t]
  int8_t tap_dh[9], tap_dw[9], tap_map[9], tap_wblk[9];
  // output pixel of grid point (h, w): (h * os + ooh, w * os + oow) of an out_H x out_W tensor (stride-2 backward-data writes one parity class per launch)
  int out_H, out_W, os, ooh, oow;
  int stages;  // ring depth = min(4, K iterations): short-K 1x1 layers take less shared memory, so more CTAs share an SM
  __nv_bfloat16* out;
  const __nv_bfloat16* y_prev;  // SiLU' epilogue: conv output of the layer that produced this conv's input, and its BN scale / shift
  const float* s_prev;
  const float* t_prev;
  // PRED epilogue: fp32 NCHW [B, c_tot, out_H, out_W], GEMM column c -> channel c_off + c, columns >= n_store (zero weight rows) dropped
  float* out_f32;
  const float* bias;
  int c_tot, c_off, n_store;
};

// D[128 pixels, BN couts] = sum over (tap, 64-channel chunk) of A[pixels, 64] * W[couts, 64]^T, bf16 x bf16 -> fp32 in registers
// (warpgroup w: pixel rows 64w..64w+63).
// SILU_BWD: the result is d(loss)/d(a_prev) with a_prev = silu(z_prev), z_prev = y_prev * s + t: the epilogue multiplies by silu'(z_prev),
// so the producer's activation gradient never makes a round trip through HBM.
// PRED: the head's prediction convs (nn.Conv2d with bias, no BatchNorm / activation): out_f32 = D + bias in fp32, stored NCHW because the
// loss reads the reference's [B, 5 + num_classes, h, w] tensor.
template <int BN, bool SILU_BWD, bool PRED = false>
__global__ void __launch_bounds__(kTThreads, 1) tconv_kernel(const __grid_constant__ TConvArgs a) {
  constexpr int A_BYTES = 128 * 128;
  constexpr int B_BYTES = BN * 128;
  constexpr int STAGE = A_BYTES + B_BYTES;
  extern __shared__ __align__(1024) uint8_t smem[];
  const int STAGES = a.stages;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE);
  uint64_t* full = bars;
  uint64_t* empty = bars + kTStagesFwd;
  float* st_s = reinterpret_cast<float*>(empty + kTStagesFwd);  // [BN] scale, [BN] shift of the producer's BN (SILU_BWD)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (warp == kTProducerWarp && lane == 0) {
    tma_prefetch_desc(&a.tmA[0]);
    tma_prefetch_desc(&a.tmB);
  }
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], kTMmaWarps);
    }
    fence_barrier_init();
  }
  const int n0 = blockIdx.y * BN;
  if (SILU_BWD) {
    for (int i = threadIdx.x; i < BN; i += kTThreads) {
      const bool in = BN != 32 || i < a.cout;  // BN = 32: the whole (16- or 32-channel) output in one tile
      st_s[i] = in ? a.s_prev[n0 + i] : 0.0f;
      st_s[BN + i] = in ? a.t_prev[n0 + i] : 0.0f;
    }
  }
  __syncthreads();

  const int mt = blockIdx.x;
  const int wt = mt % a.tiles_w, t2 = mt / a.tiles_w;
  const int ht = t2 % a.tiles_h, bt = t2 / a.tiles_h;
  const int w0 = wt * a.TW, h0 = ht * a.TH, b0 = bt * a.NB;
  // cin = 16 or 32: one chunk whose channels past cin TMA zero-fills (the 64-channel box is wider than the tensor), and the weights' K
  // blocks are padded to the chunk width with zeros (cvb_train_pack_weights)
  const int chunks = (a.cin + 63) / 64;
  const int k_iters = a.taps * chunks;

  if (warp == kTProducerWarp) {
    if (elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tap = 0; tap < a.taps; ++tap) {
        const int dh = a.tap_dh[tap], dw = a.tap_dw[tap];
        const CUtensorMap* mapA = &a.tmA[a.tap_map[tap]];
        const int kb = a.tap_wblk[tap] * chunks * 64;
        for (int ck = 0; ck < chunks; ++ck) {
          mbar_wait(&empty[stage], phase ^ 1, 100 + stage);
          mbar_expect_tx(&full[stage], A_BYTES + B_BYTES);
          uint8_t* sb = smem + stage * STAGE;
          tma_load_4d(mapA, &full[stage], sb, ck * 64, w0 + dw, h0 + dh, b0);
          tma_load_2d(&a.tmB, &full[stage], sb + A_BYTES, kb + ck * 64, n0);
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    const int wg = warp >> 2;
    float d[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) d[i] = 0.0f;
    int stage = 0, pend = -1;
    uint32_t phase = 0;
    for (int i = 0; i < k_iters; ++i) {
      mbar_wait(&full[stage], phase, 300 + stage);
      const uint32_t sa = smem_u32(smem + stage * STAGE);
      const uint64_t da = make_kmajor_desc<128>(sa + wg * (A_BYTES / 2));
      const uint64_t db = make_kmajor_desc<128>(sa + A_BYTES);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_m64k16<BN, 1, 0>(d, da + 2 * k, db + 2 * k);
      wgmma_commit();
      wgmma_wait<1>();  // the previous K chunk has been read: release its stage
      wgmma_fence_regs(d);
      if (lane == 0 && pend >= 0) mbar_arrive(&empty[pend]);
      pend = stage;
      if (++stage == STAGES) {
        stage = 0;
        phase ^= 1;
      }
    }
    wgmma_wait<0>();
    wgmma_fence_regs(d);
    // wgmma fragment: rows 64*wg + 16*(warp&3) + lane/4 (+8), columns 8*j + 2*(lane&3) (+1)
    const int r0 = 64 * wg + 16 * (warp & 3) + (lane >> 2), cq = 2 * (lane & 3);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = r0 + 8 * h;
      const int tw = row % a.TW, r2 = row / a.TW;
      const int th = r2 % a.TH, nb = r2 / a.TH;
      const int ow = w0 + tw, oh = h0 + th, ob = b0 + nb;
      if (!(ow < a.W && oh < a.H && ob < a.B)) continue;
      if (PRED) {
        const size_t plane = (size_t)a.out_H * a.out_W;
        float* ocol = a.out_f32 + ((size_t)ob * a.c_tot + a.c_off + n0) * plane + (size_t)oh * a.out_W + ow;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int c = 8 * j + cq;
          if (n0 + c < a.n_store) ocol[c * plane] = d[4 * j + 2 * h] + __ldg(a.bias + n0 + c);
          if (n0 + c + 1 < a.n_store) ocol[(c + 1) * plane] = d[4 * j + 2 * h + 1] + __ldg(a.bias + n0 + c + 1);
        }
        continue;
      }
      const size_t pix = ((size_t)ob * a.out_H + (oh * a.os + a.ooh)) * a.out_W + (ow * a.os + a.oow);
      __nv_bfloat16* orow = a.out + pix * a.cout + n0;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int c = 8 * j + cq;
        if (BN == 32 && c >= a.cout) continue;  // cout = 16: the upper half of the tile is the zero-filled weight rows
        float d0 = d[4 * j + 2 * h], d1 = d[4 * j + 2 * h + 1];
        if (SILU_BWD) {
          const float2 yf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(a.y_prev + pix * a.cout + n0 + c));
          const float z0 = fmaf(yf.x, st_s[c], st_s[BN + c]);
          const float z1 = fmaf(yf.y, st_s[c + 1], st_s[BN + c + 1]);
          const float g0 = 1.0f / (1.0f + __expf(-z0)), g1 = 1.0f / (1.0f + __expf(-z1));
          // silu'(z) = sigmoid(z) * (1 + z * (1 - sigmoid(z)))
          d0 *= g0 * fmaf(z0, 1.0f - g0, 1.0f);
          d1 *= g1 * fmaf(z1, 1.0f - g1, 1.0f);
        }
        *reinterpret_cast<__nv_bfloat162*>(orow + c) = __floats2bfloat162_rn(d0, d1);
      }
    }
  }
}

struct alignas(64) TWgradArgs {
  CUtensorMap tmX[4];  // x  {cin, W, H, B},  box {64, TW, TH, NB}; stride 2: one map per input parity class
  CUtensorMap tmD;     // dy {cout, Wo, Ho, B}, box {64, TW, TH, NB}
  int tiles_w, tiles_h, tiles_b;  // over the OUTPUT pixels (dy)
  int TW, TH, NB;
  int cin, cout, taps;
  int nblocks;  // cout / (64 * NPAN): output-channel blocks of one launch (cout = 512 runs as two 256-wide blocks, 192 as three 64-wide), folded into blockIdx.z
  int8_t tap_dh[9], tap_dw[9], tap_map[9];
  int8_t tap_idx[9];  // filter tap (dw block) of grid row blockIdx.y; `taps` = k * k is the dw layout's
  int splits;
  float* dw;  // [cout][taps][cin] fp32, accumulated with atomics (zeroed by the caller)
};

// dW^T block [128 cin rows, cout columns] of one filter tap += sum over this CTA's pixel tiles of x_tile^T * dy_tile  (K = 128 pixels per
// stage, 8 MMAs of K = 16).  Both operands are the NHWC tiles exactly as TMA lands them: MN-major (channels contiguous), 64-channel panels;
// warpgroup w owns the cin panel w (accumulator rows 64w..64w+63).
// NARROW (NPAN = 1): cout = 16 or 32; the dy panel's channels past cout are zero-filled by TMA and their columns are not stored.
template <int NPAN, bool NARROW = false>  // cout / 64
__global__ void __launch_bounds__(kTThreads, 1) twgrad_kernel(const __grid_constant__ TWgradArgs a) {
  constexpr int PANEL = 128 * 128;  // 128 pixel rows x 64 channels bf16
  constexpr int X_BYTES = 2 * PANEL;
  constexpr int D_BYTES = NPAN * PANEL;
  constexpr int STAGE = X_BYTES + D_BYTES;
  constexpr int N = NPAN * 64;
  constexpr int STAGES = NPAN == 4 ? 2 : kTStagesWg;  // 96 KB stages at cout = 256
  extern __shared__ __align__(1024) uint8_t smem[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE);
  uint64_t* full = bars;
  uint64_t* empty = bars + STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == kTProducerWarp && lane == 0) {
    tma_prefetch_desc(&a.tmX[0]);
    tma_prefetch_desc(&a.tmD);
  }
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], kTMmaWarps);
    }
    fence_barrier_init();
  }
  __syncthreads();

  const int split = blockIdx.x, ti = blockIdx.y, tap = a.tap_idx[ti], c0 = ((int)blockIdx.z / a.nblocks) * 128, n0 = ((int)blockIdx.z % a.nblocks) * N;
  const int m_pan = (a.cin - c0) >= 128 ? 2 : 1;  // valid 64-channel panels of this cin block
  const int dh = a.tap_dh[ti], dw_ = a.tap_dw[ti];
  const CUtensorMap* mapX = &a.tmX[a.tap_map[ti]];
  const int m_tiles = a.tiles_w * a.tiles_h * a.tiles_b;
  const int per = (m_tiles + a.splits - 1) / a.splits;
  const int t_begin = split * per, t_end = min(m_tiles, t_begin + per);

  if (warp == kTProducerWarp) {
    if (elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int mt = t_begin; mt < t_end; ++mt) {
        const int wt = mt % a.tiles_w, t2 = mt / a.tiles_w;
        const int ht = t2 % a.tiles_h, bt = t2 / a.tiles_h;
        const int w0 = wt * a.TW, h0 = ht * a.TH, b0 = bt * a.NB;
        mbar_wait(&empty[stage], phase ^ 1, 100 + stage);
        mbar_expect_tx(&full[stage], (uint32_t)(m_pan * PANEL + D_BYTES));
        uint8_t* sb = smem + stage * STAGE;
        for (int p = 0; p < m_pan; ++p) tma_load_4d(mapX, &full[stage], sb + p * PANEL, c0 + p * 64, w0 + dw_, h0 + dh, b0);
        for (int p = 0; p < NPAN; ++p) tma_load_4d(&a.tmD, &full[stage], sb + X_BYTES + p * PANEL, n0 + p * 64, w0, h0, b0);
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
  } else if (t_begin < t_end) {
    const int wg = warp >> 2;
    const bool active = wg < m_pan;  // (warpgroup-uniform) the second cin panel exists
    float d[N / 2];
#pragma unroll
    for (int i = 0; i < N / 2; ++i) d[i] = 0.0f;
    int stage = 0, pend = -1;
    uint32_t phase = 0;
    for (int mt = t_begin; mt < t_end; ++mt) {
      mbar_wait(&full[stage], phase, 300 + stage);
      if (active) {
        const uint32_t sa = smem_u32(smem + stage * STAGE);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 8; ++k) {  // K = 16 pixel rows = 2048 bytes per MMA
          const uint64_t da = make_mnmajor_desc_sw128(sa + wg * PANEL + k * 2048, PANEL, 1024);
          const uint64_t db = make_mnmajor_desc_sw128(sa + X_BYTES + k * 2048, PANEL, 1024);
          wgmma_m64k16<N, 1, 1>(d, da, db);
        }
        wgmma_commit();
        wgmma_wait<1>();
        wgmma_fence_regs(d);
        if (lane == 0 && pend >= 0) mbar_arrive(&empty[pend]);
        pend = stage;
      } else if (lane == 0) {
        mbar_arrive(&empty[stage]);
      }
      if (++stage == STAGES) {
        stage = 0;
        phase ^= 1;
      }
    }
    if (active) {
      wgmma_wait<0>();
      wgmma_fence_regs(d);
      // wgmma fragment: rows (cin) 64*wg + 16*(warp&3) + lane/4 (+8), columns (cout) 8*j + 2*(lane&3) (+1)
      const int r0 = 64 * wg + 16 * (warp & 3) + (lane >> 2), cq = 2 * (lane & 3);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = r0 + 8 * h;
        if (c0 + row >= a.cin) continue;
        float* base = a.dw + ((size_t)n0 * a.taps + tap) * a.cin + c0 + row;
        const size_t cstride = (size_t)a.taps * a.cin;
#pragma unroll
        for (int j = 0; j < N / 8; ++j) {
          const int c = 8 * j + cq;
          if (NARROW && c >= a.cout) continue;
          atomicAdd(base + (size_t)c * cstride, d[4 * j + 2 * h]);
          atomicAdd(base + (size_t)(c + 1) * cstride, d[4 * j + 2 * h + 1]);
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ BatchNorm + SiLU element-wise passes
// NHWC bf16, C a multiple of 8.  A thread owns one 8-channel vector column and walks pixels; per-channel partial sums are combined in
// shared memory, then one atomicAdd per channel and CTA.
constexpr int kEwThreads = 256;

__device__ __forceinline__ void bf16x8_to_float(const uint4& u, float (&f)[8]) {
  const __nv_bfloat162* p = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = __bfloat1622float2(p[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ uint4 float_to_bf16x8(const float (&f)[8]) {
  uint4 u;
  __nv_bfloat162* p = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) p[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  return u;
}

// Per-channel reductions over pixels: a CTA owns a contiguous pixel range, thread (v, pl) = (8-channel vector, pixel lane) accumulates in
// registers, the pixel lanes are combined through shared memory ([lane][2C] partials, no atomics) and 2C global atomicAdds leave the CTA.
constexpr int kRedSmemFloats = kEwThreads * 16;  // np * 2C == 256 * 16 for every C

__device__ __forceinline__ void red_finish(float (&a1)[8], float (&a2)[8], int v, int pl, int np, bool active, int C, float* s_part, float* __restrict__ sums) {
  if (active) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      s_part[pl * 2 * C + v * 8 + i] = a1[i];
      s_part[pl * 2 * C + C + v * 8 + i] = a2[i];
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < 2 * C; c += kEwThreads) {
    float t = 0.0f;
    for (int l = 0; l < np; ++l) t += s_part[l * 2 * C + c];
    atomicAdd(&sums[c], t);
  }
}

// sums[c] += sum_p (y[p][c] - y[0][c]), sums[C + c] += sum_p (y[p][c] - y[0][c])^2
// The pivot y[0][c] (a sample of the channel) keeps the sums at the scale of the channel's spread, not of its mean: E[y^2] - mean^2 in fp32
// loses (mean / std)^2 times the accumulation error, which a channel with mean = 100 * std turns into a 1e-3 error of rstd.
__global__ void __launch_bounds__(kEwThreads) bn_stats_kernel(const __nv_bfloat16* __restrict__ y, long long npix, int C, float* __restrict__ sums) {
  __shared__ float s_part[kRedSmemFloats];
  const int cv = C / 8;
  const int v = threadIdx.x % cv;
  const int pl = threadIdx.x / cv, np = kEwThreads / cv;
  const bool active = pl < np;
  const long long chunk = (npix + gridDim.x - 1) / gridDim.x;
  const long long p0 = (long long)blockIdx.x * chunk, p1 = min(npix, p0 + chunk);
  float a1[8], a2[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) a1[i] = a2[i] = 0.0f;
  if (active) {
    float k[8];
    bf16x8_to_float(__ldg(reinterpret_cast<const uint4*>(y) + v), k);
    long long p = p0 + pl;
    for (; p + np < p1; p += 2 * np) {  // two independent 16-byte loads in flight
      float f[8], h[8];
      const uint4 u0 = __ldg(reinterpret_cast<const uint4*>(y + p * C) + v);
      const uint4 u1 = __ldg(reinterpret_cast<const uint4*>(y + (p + np) * C) + v);
      bf16x8_to_float(u0, f);
      bf16x8_to_float(u1, h);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float d0 = f[i] - k[i], d1 = h[i] - k[i];
        a1[i] += d0 + d1;
        a2[i] = fmaf(d0, d0, fmaf(d1, d1, a2[i]));
      }
    }
    if (p < p1) {
      float f[8];
      bf16x8_to_float(__ldg(reinterpret_cast<const uint4*>(y + p * C) + v), f);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float d0 = f[i] - k[i];
        a1[i] += d0;
        a2[i] = fmaf(d0, d0, a2[i]);
      }
    }
  }
  red_finish(a1, a2, v, pl, np, active, C, s_part, sums);
}

// channel c's batch mean and biased variance over n pixels -> mean, rstd, folded scale / shift; running statistics updated like
// nn.BatchNorm2d (unbiased variance, momentum).  Shared by the local (bn_finalize_kernel) and the cross-rank (bn_merge_kernel) statistics.
__device__ __forceinline__ void bn_finalize_channel(int c, int C, double mean, double var, double n, const float* __restrict__ gamma,
                                                    const float* __restrict__ beta, float eps, float momentum, float* __restrict__ running_mean,
                                                    float* __restrict__ running_var, float* __restrict__ stat) {
  if (var < 0.0) var = 0.0;
  const float rstd = (float)(1.0 / sqrt(var + (double)eps));
  const float s = gamma[c] * rstd;
  stat[c] = (float)mean;
  stat[C + c] = rstd;
  stat[2 * C + c] = s;
  stat[3 * C + c] = beta[c] - (float)mean * s;
  if (running_mean != nullptr) {
    running_mean[c] = (1.0f - momentum) * running_mean[c] + momentum * (float)mean;
    running_var[c] = (1.0f - momentum) * running_var[c] + momentum * (float)(var * n / (n > 1.0 ? n - 1.0 : 1.0));
  }
}

// batch statistics of this device's pixels (bn_stats_kernel's pivoted sums) -> stat [4][C], running statistics
__global__ void bn_finalize_kernel(const float* __restrict__ sums, const __nv_bfloat16* __restrict__ y, long long npix, int C, const float* __restrict__ gamma,
                                   const float* __restrict__ beta, float eps, float momentum, float* __restrict__ running_mean, float* __restrict__ running_var,
                                   float* __restrict__ stat /* [4][C]: mean, rstd, scale, shift */) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double n = (double)npix;
  const double d1 = (double)sums[c] / n;  // mean - pivot
  const double mean = (double)__bfloat162float(y[c]) + d1;
  const double var = (double)sums[C + c] / n - d1 * d1;
  bn_finalize_channel(c, C, mean, var, n, gamma, beta, eps, momentum, running_mean, running_var, stat);
}

// Cross-rank (SyncBatchNorm) statistics.  Every rank's pivot y[0][c] is a different sample, so the pivoted sums of two ranks do not add;
// each rank turns its sums into a record of (count, mean, M2 = sum of squared deviations from its own mean), which merge exactly.
// Record layout, fp64 [2C + 1]: mean[C], M2[C], count.
__global__ void bn_partial_kernel(const float* __restrict__ sums, const __nv_bfloat16* __restrict__ y, long long npix, int C, double* __restrict__ rec) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double n = (double)npix;
  const double s1 = (double)sums[c];
  const double d1 = s1 / n;  // mean - pivot
  rec[c] = (double)__bfloat162float(y[c]) + d1;
  const double m2 = (double)sums[C + c] - s1 * d1;  // = n * (S2 / n - d1^2), the variance bn_finalize_kernel takes, times n
  rec[C + c] = m2 > 0.0 ? m2 : 0.0;
  if (c == 0) rec[2 * C] = n;
}

// records [world][2C + 1] (as all_gather lays them out) -> Chan's pairwise merge in rank order, in fp64, so every rank computes the same bits
// -> stat [4][C] and running statistics as bn_finalize_kernel; *count = the global pixel count, for the backward's 1 / N.
__global__ void bn_merge_kernel(const double* __restrict__ recs, int world, int C, const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                float momentum, float* __restrict__ running_mean, float* __restrict__ running_var, float* __restrict__ stat,
                                double* __restrict__ count) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const long long len = 2 * (long long)C + 1;
  double n = recs[2 * C], mean = recs[c], m2 = recs[C + c];
  for (int r = 1; r < world; ++r) {
    const double* rb = recs + r * len;
    const double nb = rb[2 * C], nab = n + nb;
    const double delta = rb[c] - mean;
    mean += delta * (nb / nab);
    m2 += rb[C + c] + delta * delta * (n * nb / nab);
    n = nab;
  }
  bn_finalize_channel(c, C, mean, m2 / n, n, gamma, beta, eps, momentum, running_mean, running_var, stat);
  if (c == 0) *count = n;
}

__device__ __forceinline__ float silu_grad(float z) {
  const float g = 1.0f / (1.0f + __expf(-z));
  return g * fmaf(z, 1.0f - g, 1.0f);
}

// The activation after a training BatchNorm: SiLU (YOLOX, YOLOv5, the YOLOv6 head) or ReLU (the YOLOv6 backbone and neck).  The ReLU
// gradient passes where z > 0, torch's rule; z is the same fp32 fmaf(y, scale, shift) in the forward and both backward passes.
enum : int { kActSilu = 0, kActRelu = 1 };
template <int ACT>
__device__ __forceinline__ float act_fwd(float z) {
  return ACT == kActRelu ? fmaxf(z, 0.0f) : z / (1.0f + __expf(-z));
}
template <int ACT>
__device__ __forceinline__ float act_grad(float z) {
  return ACT == kActRelu ? (z > 0.0f ? 1.0f : 0.0f) : silu_grad(z);
}

// a = act(y * scale + shift)
template <int ACT>
__global__ void __launch_bounds__(kEwThreads) bn_act_fwd_kernel(const __nv_bfloat16* __restrict__ y, long long nvec, int C, const float* __restrict__ stat,
                                                                 __nv_bfloat16* __restrict__ out) {
  const int cv = C / 8;
  const long long stride = (long long)gridDim.x * kEwThreads;
  for (long long i = (long long)blockIdx.x * kEwThreads + threadIdx.x; i < nvec; i += 2 * stride) {
    const long long i2 = i + stride;
    const bool two = i2 < nvec;
    const uint4 u0 = __ldg(reinterpret_cast<const uint4*>(y) + i);
    const uint4 u1 = two ? __ldg(reinterpret_cast<const uint4*>(y) + i2) : u0;  // two independent 16-byte loads in flight
    {
      const int c0 = (int)(i % cv) * 8;
      float f[8];
      bf16x8_to_float(u0, f);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float z = fmaf(f[k], __ldg(stat + 2 * C + c0 + k), __ldg(stat + 3 * C + c0 + k));
        f[k] = act_fwd<ACT>(z);
      }
      reinterpret_cast<uint4*>(out)[i] = float_to_bf16x8(f);
    }
    if (two) {
      const int c0 = (int)(i2 % cv) * 8;
      float f[8];
      bf16x8_to_float(u1, f);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float z = fmaf(f[k], __ldg(stat + 2 * C + c0 + k), __ldg(stat + 3 * C + c0 + k));
        f[k] = act_fwd<ACT>(z);
      }
      reinterpret_cast<uint4*>(out)[i2] = float_to_bf16x8(f);
    }
  }
}

// sums[c] += sum_p dz, sums[C + c] += sum_p dz * xhat   (dz = g * act'(z) when `g` is d(loss)/d(a); dz = g when g_is_dz)
template <int ACT>
__global__ void __launch_bounds__(kEwThreads) bn_act_bwd_reduce_kernel(const __nv_bfloat16* __restrict__ g, const __nv_bfloat16* __restrict__ y, long long npix,
                                                                        int C, const float* __restrict__ stat, int g_is_dz, float* __restrict__ sums) {
  __shared__ float s_part[kRedSmemFloats];
  const int cv = C / 8;
  const int v = threadIdx.x % cv;
  const int pl = threadIdx.x / cv, np = kEwThreads / cv;
  const bool active = pl < np;
  const long long chunk = (npix + gridDim.x - 1) / gridDim.x;
  const long long p0 = (long long)blockIdx.x * chunk, p1 = min(npix, p0 + chunk);
  float a1[8], a2[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) a1[i] = a2[i] = 0.0f;
  if (active) {
    float mean[8], rstd[8], sc[8], sh[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      mean[i] = stat[v * 8 + i];
      rstd[i] = stat[C + v * 8 + i];
      sc[i] = stat[2 * C + v * 8 + i];
      sh[i] = stat[3 * C + v * 8 + i];
    }
    for (long long p = p0 + pl; p < p1; p += np) {
      float fy[8], fg[8];
      const uint4 uy = __ldg(reinterpret_cast<const uint4*>(y + p * C) + v);
      const uint4 ug = __ldg(reinterpret_cast<const uint4*>(g + p * C) + v);
      bf16x8_to_float(uy, fy);
      bf16x8_to_float(ug, fg);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float dz = g_is_dz ? fg[i] : fg[i] * act_grad<ACT>(fmaf(fy[i], sc[i], sh[i]));
        a1[i] += dz;
        a2[i] = fmaf(dz, (fy[i] - mean[i]) * rstd[i], a2[i]);
      }
    }
  }
  red_finish(a1, a2, v, pl, np, active, C, s_part, sums);
}

// dy = gamma * rstd * (dz - sum_dz / N - xhat * sum_dzx / N);  1 / N = inv_n, or (DEV_COUNT: N over every rank) 1 / *count, read on the device
template <int ACT, bool DEV_COUNT>
__global__ void __launch_bounds__(kEwThreads) bn_act_bwd_apply_kernel(const __nv_bfloat16* __restrict__ g, const __nv_bfloat16* __restrict__ y, long long nvec, int C,
                                                                       const float* __restrict__ stat, const float* __restrict__ gamma, const float* __restrict__ sums,
                                                                       float inv_n, const double* __restrict__ count, int g_is_dz, __nv_bfloat16* __restrict__ dy) {
  if (DEV_COUNT) inv_n = (float)(1.0 / __ldg(count));
  const int cv = C / 8;
  const long long stride = (long long)gridDim.x * kEwThreads;
  for (long long i = (long long)blockIdx.x * kEwThreads + threadIdx.x; i < nvec; i += 2 * stride) {
    const long long i2 = i + stride;
    const bool two = i2 < nvec;
    // four independent 16-byte loads in flight
    const uint4 uy0 = __ldg(reinterpret_cast<const uint4*>(y) + i), ug0 = __ldg(reinterpret_cast<const uint4*>(g) + i);
    const uint4 uy1 = two ? __ldg(reinterpret_cast<const uint4*>(y) + i2) : uy0, ug1 = two ? __ldg(reinterpret_cast<const uint4*>(g) + i2) : ug0;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (h == 1 && !two) break;
      const long long ii = h ? i2 : i;
      const int c0 = (int)(ii % cv) * 8;
      float fy[8], fg[8];
      bf16x8_to_float(h ? uy1 : uy0, fy);
      bf16x8_to_float(h ? ug1 : ug0, fg);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int c = c0 + k;
        const float mean = __ldg(stat + c), rstd = __ldg(stat + C + c);
        const float dz = g_is_dz ? fg[k] : fg[k] * act_grad<ACT>(fmaf(fy[k], __ldg(stat + 2 * C + c), __ldg(stat + 3 * C + c)));
        const float xhat = (fy[k] - mean) * rstd;
        fg[k] = __ldg(gamma + c) * rstd * (dz - __ldg(sums + c) * inv_n - xhat * __ldg(sums + C + c) * inv_n);
      }
      reinterpret_cast<uint4*>(dy)[ii] = float_to_bf16x8(fg);
    }
  }
}

// ------------------------------------------------------------------------------------------------ Focus stem and SPPF pooling
// Focus (src/models/modules/yolo_modules.py:19-37): fp32 NCHW [B,3,H,W] -> bf16 NHWC [B,H/2,W/2,16], channel 3 * patch + c in the reference's
// patch order tl, bl, tr, br (patch = 2 * dx + dy), channels 12..15 zero: the 12 -> cout stem conv then runs as a 16-channel conv whose
// weight is the reference's, zero-padded.  One thread per output pixel; a float2 load holds the dx = 0 / 1 pair of one (c, dy) row.
__global__ void __launch_bounds__(kEwThreads) focus_s2d_kernel(const float* __restrict__ img, int B, int H, int W, __nv_bfloat16* __restrict__ out) {
  const int Ho = H / 2, Wo = W / 2;
  const long long n = (long long)B * Ho * Wo;
  for (long long p = blockIdx.x * (long long)kEwThreads + threadIdx.x; p < n; p += (long long)gridDim.x * kEwThreads) {
    const int ow = (int)(p % Wo);
    const long long t = p / Wo;
    const int oh = (int)(t % Ho), b = (int)(t / Ho);
    float lo[8], hi[8];
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
      for (int dy = 0; dy < 2; ++dy) {
        const float2 v = __ldg(reinterpret_cast<const float2*>(img + (((size_t)b * 3 + c) * H + 2 * oh + dy) * W + 2 * ow));
        const int c0 = 3 * dy + c, c1 = 3 * (2 + dy) + c;  // (dx = 0: patch dy; dx = 1: patch 2 + dy)
        if (c0 < 8) lo[c0] = v.x; else hi[c0 - 8] = v.x;
        if (c1 < 8) lo[c1] = v.y; else hi[c1 - 8] = v.y;
      }
#pragma unroll
    for (int i = 4; i < 8; ++i) hi[i] = 0.0f;
    uint4* o = reinterpret_cast<uint4*>(out + p * 16);
    o[0] = float_to_bf16x8(lo);
    o[1] = float_to_bf16x8(hi);
  }
}

// SPPF pooling (yolo_modules.py:165-194, kernel_sizes (5, 9, 13), stride 1, padding k // 2, the three pools in parallel on conv1's output):
// a [B,H,W,C] -> cat [B,H,W,4C] = [a | mp5 | mp9 | mp13] (conv2's input, no separate concat) and, per pool and element, the winner's
// row-major offset inside its window, idx [3][B*H*W][C] uint8 (13 * 13 = 169 offsets).  The windows are nested and centred on the same
// pixel, so one row-major scan of the 13 x 13 neighbourhood serves all three; a value replaces the running maximum only if it is strictly
// greater (or NaN), so the first maximal element in row-major window order wins -- the rule of PyTorch's max_pool2d, which decides where the
// backward routes a tie.  Positions outside the map are skipped (the padding never wins: the centre is always inside).
// Thread = one 8-channel vector of one pixel.
__global__ void __launch_bounds__(kEwThreads) spp_pool_fwd_kernel(const __nv_bfloat16* __restrict__ a, int B, int H, int W, int C, __nv_bfloat16* __restrict__ cat,
                                                                  uint8_t* __restrict__ idx) {
  const int cv = C / 8;
  const long long npix = (long long)B * H * W, n = npix * cv;
  for (long long i = blockIdx.x * (long long)kEwThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kEwThreads) {
    const int v = (int)(i % cv);
    const long long p = i / cv;
    const int w = (int)(p % W);
    const long long t = p / W;
    const int h = (int)(t % H);
    const long long img = (t / H) * H * W;
    float m[3][8];
    int k[3][8];
#pragma unroll
    for (int s = 0; s < 3; ++s)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        m[s][j] = -INFINITY;
        k[s][j] = 0;
      }
    for (int dy = -6; dy <= 6; ++dy) {
      const int y = h + dy;
      if (y < 0 || y >= H) continue;
      for (int dx = -6; dx <= 6; ++dx) {
        const int x = w + dx;
        if (x < 0 || x >= W) continue;
        float f[8];
        bf16x8_to_float(__ldg(reinterpret_cast<const uint4*>(a + ((img + (long long)y * W + x) * C)) + v), f);
        const bool in9 = dy >= -4 && dy <= 4 && dx >= -4 && dx <= 4, in5 = dy >= -2 && dy <= 2 && dx >= -2 && dx <= 2;
        const int o13 = (dy + 6) * 13 + dx + 6, o9 = (dy + 4) * 9 + dx + 4, o5 = (dy + 2) * 5 + dx + 2;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const bool nan = f[j] != f[j];
          if (in5 && (f[j] > m[0][j] || nan)) { m[0][j] = f[j]; k[0][j] = o5; }
          if (in9 && (f[j] > m[1][j] || nan)) { m[1][j] = f[j]; k[1][j] = o9; }
          if (f[j] > m[2][j] || nan) { m[2][j] = f[j]; k[2][j] = o13; }
        }
      }
    }
    uint4* crow = reinterpret_cast<uint4*>(cat + p * 4 * C) + v;
    crow[0] = __ldg(reinterpret_cast<const uint4*>(a + p * C) + v);
#pragma unroll
    for (int s = 0; s < 3; ++s) {
      crow[(s + 1) * cv] = float_to_bf16x8(m[s]);  // (bf16 values: the conversion is exact)
      if (idx == nullptr) continue;  // (the chained SPPF takes the values only: sppf_chain_idx_kernel records its winners)
      uint2 u;
      u.x = (uint32_t)k[s][0] | ((uint32_t)k[s][1] << 8) | ((uint32_t)k[s][2] << 16) | ((uint32_t)k[s][3] << 24);
      u.y = (uint32_t)k[s][4] | ((uint32_t)k[s][5] << 8) | ((uint32_t)k[s][6] << 16) | ((uint32_t)k[s][7] << 24);
      reinterpret_cast<uint2*>(idx + ((long long)s * npix + p) * C)[v] = u;
    }
  }
}

// da = g[:, :C] + sum over pools s and the windows q that contain p and chose p: g[q][(s + 1) C + c] -- a gather in a fixed order (q row-major,
// then s), summed in fp32 and rounded to bf16 once: bitwise reproducible, no atomics.
__global__ void __launch_bounds__(kEwThreads) spp_pool_bwd_kernel(const __nv_bfloat16* __restrict__ g, const uint8_t* __restrict__ idx, int B, int H, int W, int C,
                                                                  __nv_bfloat16* __restrict__ da) {
  const int cv = C / 8;
  const long long npix = (long long)B * H * W, n = npix * cv;
  for (long long i = blockIdx.x * (long long)kEwThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kEwThreads) {
    const int v = (int)(i % cv);
    const long long p = i / cv;
    const int w = (int)(p % W);
    const long long t = p / W;
    const int h = (int)(t % H);
    const long long img = (t / H) * H * W;
    float acc[8];
    bf16x8_to_float(__ldg(reinterpret_cast<const uint4*>(g + p * 4 * C) + v), acc);
    for (int ey = -6; ey <= 6; ++ey) {  // q = (h + ey, w + ex): p sits at (-ey, -ex) from q's centre
      const int y = h + ey;
      if (y < 0 || y >= H) continue;
      for (int ex = -6; ex <= 6; ++ex) {
        const int x = w + ex;
        if (x < 0 || x >= W) continue;
        const long long q = img + (long long)y * W + x;
#pragma unroll
        for (int s = 0; s < 3; ++s) {
          const int r = 2 + 2 * s, kk = 2 * r + 1;  // 5, 9, 13
          if (ey < -r || ey > r || ex < -r || ex > r) continue;
          const uint32_t off = (uint32_t)((r - ey) * kk + (r - ex));
          const uint2 u = __ldg(reinterpret_cast<const uint2*>(idx + ((long long)s * npix + q) * C) + v);
          const uint32_t want = off * 0x01010101u;
          // bytes of u equal to `off`: one bit per channel (a byte of x ^ want is zero)
          uint32_t hit = 0;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            hit |= ((((u.x ^ want) >> (8 * j)) & 0xffu) == 0u ? 1u : 0u) << j;
            hit |= ((((u.y ^ want) >> (8 * j)) & 0xffu) == 0u ? 1u : 0u) << (4 + j);
          }
          if (hit == 0) continue;
          float f[8];
          bf16x8_to_float(__ldg(reinterpret_cast<const uint4*>(g + q * 4 * C + (s + 1) * C) + v), f);
#pragma unroll
          for (int j = 0; j < 8; ++j)
            if (hit & (1u << j)) acc[j] += f[j];
        }
      }
    }
    reinterpret_cast<uint4*>(da + p * C)[v] = float_to_bf16x8(acc);
  }
}

// Chained SPPF (yolo_modules.py:165-194 with kernel_sizes = 5): y1 = mp5(x), y2 = mp5(y1), y3 = mp5(y2).  The values are those of the
// parallel 5 / 9 / 13 pools (spp_pool_fwd_kernel writes cat = [x | y1 | y2 | y3]), but autograd through the chain routes each stage's
// gradient to the winner of the 5 x 5 window of that stage's own input, which on ties is not the parallel pools' winner.  idx [3][B*H*W][C]
// uint8: per stage s, the row-major offset (0..24) in the window over cat slice s of its first maximum (NaN wins; the window starts at its
// first in-map element, as in max_pool2d).  Thread = one (pixel, channel).
__global__ void __launch_bounds__(kEwThreads) sppf_chain_idx_kernel(const __nv_bfloat16* __restrict__ cat, int B, int H, int W, int C, uint8_t* __restrict__ idx) {
  const long long npix = (long long)B * H * W, n = npix * C;
  for (long long i = blockIdx.x * (long long)kEwThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kEwThreads) {
    const int c = (int)(i % C);
    const long long p = i / C;
    const int w = (int)(p % W);
    const long long t = p / W;
    const int h = (int)(t % H);
    const long long img = (t / H) * H * W;
    for (int s = 0; s < 3; ++s) {
      float m = -INFINITY;
      int k = (max(-h, -2) + 2) * 5 + max(-w, -2) + 2;
      for (int dy = -2; dy <= 2; ++dy) {
        const int y = h + dy;
        if (y < 0 || y >= H) continue;
        for (int dx = -2; dx <= 2; ++dx) {
          const int x = w + dx;
          if (x < 0 || x >= W) continue;
          const float f = __bfloat162float(cat[(img + (long long)y * W + x) * 4 * C + s * C + c]);
          if (f > m || f != f) { m = f; k = (dy + 2) * 5 + dx + 2; }
        }
      }
      idx[(s * npix + p) * C + c] = (uint8_t)k;
    }
  }
}

// One backward stage of the chain: D_s = g[..., s C + c] + the D_{s+1} of every q in the 5 x 5 around p whose stage-s window chose p, in
// row-major q order (D_3 = g[..., 3C + c]).  d_next: fp32 D_{s+1}, or nullptr for s = 2; the result goes to d_out (fp32) or, for s = 0, to
// da (bf16, rounded once).  A deterministic gather: no atomics.
__global__ void __launch_bounds__(kEwThreads) sppf_chain_bwd_kernel(const __nv_bfloat16* __restrict__ g, const uint8_t* __restrict__ idx, int s,
                                                                    const float* __restrict__ d_next, float* __restrict__ d_out, __nv_bfloat16* __restrict__ da,
                                                                    int B, int H, int W, int C) {
  const long long npix = (long long)B * H * W, n = npix * C;
  const uint8_t* is = idx + s * n;
  for (long long i = blockIdx.x * (long long)kEwThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kEwThreads) {
    const int c = (int)(i % C);
    const long long p = i / C;
    const int w = (int)(p % W);
    const long long t = p / W;
    const int h = (int)(t % H);
    const long long img = (t / H) * H * W;
    float acc = __bfloat162float(g[p * 4 * C + s * C + c]);
    for (int ey = -2; ey <= 2; ++ey) {  // q = (h + ey, w + ex): p sits at (-ey, -ex) from q's centre
      const int y = h + ey;
      if (y < 0 || y >= H) continue;
      for (int ex = -2; ex <= 2; ++ex) {
        const int x = w + ex;
        if (x < 0 || x >= W) continue;
        const long long q = img + (long long)y * W + x;
        if (is[q * C + c] != (uint8_t)((2 - ey) * 5 + (2 - ex))) continue;
        acc += d_next ? d_next[q * C + c] : __bfloat162float(g[q * 4 * C + (s + 1) * C + c]);
      }
    }
    if (d_out) d_out[i] = acc;
    else da[i] = __float2bfloat16_rn(acc);
  }
}

// ------------------------------------------------------------------------------------------------ YOLOX neck and head
// Neck top-down path (src/models/necks/yolox_neck.py:52-62): cat [B,2h,2w,Ca+Cb] = [nearest_up2(a) | b].  Thread = one 16-byte vector of cat.
__global__ void __launch_bounds__(kEwThreads) upsample_cat_fwd_kernel(const __nv_bfloat16* __restrict__ a, int B, int h, int w, int Ca,
                                                                      const __nv_bfloat16* __restrict__ b, int Cb, __nv_bfloat16* __restrict__ cat) {
  const int cva = Ca / 8, cvb = Cb / 8, cv = cva + cvb, W2 = 2 * w;
  const long long n = (long long)B * 4 * h * w * cv;
  for (long long i = blockIdx.x * (long long)kEwThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kEwThreads) {
    const int v = (int)(i % cv);
    const long long p = i / cv;
    const int x = (int)(p % W2);
    const long long t = p / W2;
    const int y = (int)(t % (2 * h));
    const long long img = t / (2 * h);
    reinterpret_cast<uint4*>(cat)[i] = v < cva ? __ldg(reinterpret_cast<const uint4*>(a + ((img * h + y / 2) * w + x / 2) * Ca) + v)
                                               : __ldg(reinterpret_cast<const uint4*>(b + p * Cb) + (v - cva));
  }
}

// g = d(loss)/d(cat) -> da [B,h,w,Ca] = the 2x2 sum of g[..., :Ca] (fp32, in the fixed order (0,0), (0,1), (1,0), (1,1), one bf16 rounding)
// and db [B,2h,2w,Cb] = g[..., Ca:].  Items [0, na) are da vectors, the rest db vectors; no atomics, so bitwise reproducible.
__global__ void __launch_bounds__(kEwThreads) upsample_cat_bwd_kernel(const __nv_bfloat16* __restrict__ g, int B, int h, int w, int Ca, int Cb,
                                                                      __nv_bfloat16* __restrict__ da, __nv_bfloat16* __restrict__ db) {
  const int cva = Ca / 8, cvb = Cb / 8, cv = cva + cvb, W2 = 2 * w;
  const long long na = (long long)B * h * w * cva, n = na + (long long)B * 4 * h * w * cvb;
  for (long long i = blockIdx.x * (long long)kEwThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kEwThreads) {
    if (i < na) {
      const int v = (int)(i % cva);
      const long long p = i / cva;
      const int x = (int)(p % w);
      const long long t = p / w;
      const int y = (int)(t % h);
      const long long img = t / h;
      float acc[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = 0.0f;
#pragma unroll
      for (int dy = 0; dy < 2; ++dy)
#pragma unroll
        for (int dx = 0; dx < 2; ++dx) {
          const long long q = (img * 2 * h + 2 * y + dy) * W2 + 2 * x + dx;
          float f[8];
          bf16x8_to_float(__ldg(reinterpret_cast<const uint4*>(g + q * 8 * cv) + v), f);
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[j] += f[j];
        }
      reinterpret_cast<uint4*>(da)[i] = float_to_bf16x8(acc);
    } else {
      const long long k = i - na;
      const int v = (int)(k % cvb);
      const long long p = k / cvb;
      reinterpret_cast<uint4*>(db)[k] = __ldg(reinterpret_cast<const uint4*>(g + p * 8 * cv) + cva + v);
    }
  }
}

// Prediction-conv backward, the gradient half: the loss's fp32 NCHW gradient of output channels [c_off, c_off + cout) -> the bf16 NHWC operand
// dy [B,h,w,cout_pad] of backward-data / backward-weight, channels past cout zero.  Item i = v * npix + p (vector-major), so a warp reads 32
// consecutive pixels of one channel plane.
__global__ void __launch_bounds__(kEwThreads) pred_grad_nhwc_kernel(const float* __restrict__ g, int B, int c_tot, long long hw, int c_off, int cout, int cout_pad,
                                                                    __nv_bfloat16* __restrict__ dy) {
  const int cv = cout_pad / 8;
  const long long npix = (long long)B * hw, n = npix * cv;
  for (long long i = blockIdx.x * (long long)kEwThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kEwThreads) {
    const int v = (int)(i / npix);
    const long long p = i % npix;
    const long long b = p / hw, q = p % hw;
    const float* col = g + (b * c_tot + c_off) * hw + q;
    float f[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = 8 * v + j;
      f[j] = c < cout ? __ldg(col + c * hw) : 0.0f;
    }
    reinterpret_cast<uint4*>(dy + p * cout_pad)[v] = float_to_bf16x8(f);
  }
}

// ... and the bias half: dbias[c] = sum over images and pixels of g[:, c_off + c], one CTA per channel, thread partial sums combined by a
// fixed shared-memory tree (deterministic, no atomics).
__global__ void __launch_bounds__(kEwThreads) pred_bias_grad_kernel(const float* __restrict__ g, int B, int c_tot, long long hw, int c_off, float* __restrict__ dbias) {
  __shared__ float part[kEwThreads];
  const int c = blockIdx.x;
  float acc = 0.0f;
  for (int b = 0; b < B; ++b) {
    const float* plane = g + ((long long)b * c_tot + c_off + c) * hw;
    for (long long q = threadIdx.x; q < hw; q += kEwThreads) acc += __ldg(plane + q);
  }
  part[threadIdx.x] = acc;
  __syncthreads();
  for (int s = kEwThreads / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) part[threadIdx.x] += part[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) dbias[c] = part[0];
}

// ------------------------------------------------------------------------------------------------ YOLOv6: RepVGG blocks, BiFusion upsample
// RepVGG block in training form (src/models/modules/yolo_modules.py:268-327): a = relu(bn3(y3) + bn1(y1) [+ bnid(x)]), each BatchNorm with
// its own batch statistics (stat [4][C] of cvb_train_bn_stats).  ID: the identity branch exists (cin == cout, stride 1).  The sum is
// (z3 + z1) + zid in fp32, every z_b = fmaf(y_b, scale_b, shift_b).  One item = one 8-channel vector.
struct RepvggStats {
  const float* s3;
  const float* s1;
  const float* sid;
};

template <bool ID>
__global__ void __launch_bounds__(kEwThreads) repvgg_fwd_kernel(const __nv_bfloat16* __restrict__ y3, const __nv_bfloat16* __restrict__ y1,
                                                                const __nv_bfloat16* __restrict__ x, long long nvec, int C, RepvggStats st,
                                                                __nv_bfloat16* __restrict__ out) {
  const int cv = C / 8;
  for (long long i = blockIdx.x * (long long)kEwThreads + threadIdx.x; i < nvec; i += (long long)gridDim.x * kEwThreads) {
    const int c0 = (int)(i % cv) * 8;
    float f3[8], f1[8], fx[8];
    bf16x8_to_float(__ldg(reinterpret_cast<const uint4*>(y3) + i), f3);
    bf16x8_to_float(__ldg(reinterpret_cast<const uint4*>(y1) + i), f1);
    if (ID) bf16x8_to_float(__ldg(reinterpret_cast<const uint4*>(x) + i), fx);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int c = c0 + k;
      float z = fmaf(f3[k], __ldg(st.s3 + 2 * C + c), __ldg(st.s3 + 3 * C + c)) + fmaf(f1[k], __ldg(st.s1 + 2 * C + c), __ldg(st.s1 + 3 * C + c));
      if (ID) z += fmaf(fx[k], __ldg(st.sid + 2 * C + c), __ldg(st.sid + 3 * C + c));
      f3[k] = act_fwd<kActRelu>(z);
    }
    reinterpret_cast<uint4*>(out)[i] = float_to_bf16x8(f3);
  }
}

// Backward, reduce half: dz = g * [a > 0] (a: the forward's saved output) is every branch's BatchNorm-output gradient, so
// sums [4][C] = (sum dz = each branch's dbeta, sum dz * xhat3, sum dz * xhat1, sum dz * xhatid = the three dgammas).
template <bool ID>
__global__ void __launch_bounds__(kEwThreads) repvgg_bwd_reduce_kernel(const __nv_bfloat16* __restrict__ g, const __nv_bfloat16* __restrict__ a,
                                                                       const __nv_bfloat16* __restrict__ y3, const __nv_bfloat16* __restrict__ y1,
                                                                       const __nv_bfloat16* __restrict__ x, long long npix, int C, RepvggStats st,
                                                                       float* __restrict__ sums) {
  __shared__ float s_part[kRedSmemFloats];
  const int cv = C / 8;
  const int v = threadIdx.x % cv;
  const int pl = threadIdx.x / cv, np = kEwThreads / cv;
  const bool active = pl < np;
  const long long chunk = (npix + gridDim.x - 1) / gridDim.x;
  const long long p0 = (long long)blockIdx.x * chunk, p1 = min(npix, p0 + chunk);
  float sdz[8], s3[8], s1[8], sid[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) sdz[i] = s3[i] = s1[i] = sid[i] = 0.0f;
  if (active) {
    for (long long p = p0 + pl; p < p1; p += np) {
      const long long off = p * C;
      float fg[8], fa[8], f3[8], f1[8], fx[8];
      bf16x8_to_float(__ldg(reinterpret_cast<const uint4*>(g + off) + v), fg);
      bf16x8_to_float(__ldg(reinterpret_cast<const uint4*>(a + off) + v), fa);
      bf16x8_to_float(__ldg(reinterpret_cast<const uint4*>(y3 + off) + v), f3);
      bf16x8_to_float(__ldg(reinterpret_cast<const uint4*>(y1 + off) + v), f1);
      if (ID) bf16x8_to_float(__ldg(reinterpret_cast<const uint4*>(x + off) + v), fx);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int c = v * 8 + i;
        const float dz = fa[i] > 0.0f ? fg[i] : 0.0f;
        sdz[i] += dz;
        s3[i] = fmaf(dz, (f3[i] - __ldg(st.s3 + c)) * __ldg(st.s3 + C + c), s3[i]);
        s1[i] = fmaf(dz, (f1[i] - __ldg(st.s1 + c)) * __ldg(st.s1 + C + c), s1[i]);
        if (ID) sid[i] = fmaf(dz, (fx[i] - __ldg(st.sid + c)) * __ldg(st.sid + C + c), sid[i]);
      }
    }
  }
  red_finish(sdz, s3, v, pl, np, active, C, s_part, sums);
  __syncthreads();  // (s_part is reused)
  red_finish(s1, sid, v, pl, np, active, C, s_part, sums + 2 * C);
}

// ... apply half: dy_b = gamma_b * rstd_b * (dz - sum dz / N - xhat_b * sum(dz * xhat_b) / N) for b = 3x3, 1x1 and (ID) the identity
// branch, whose dy is its contribution to d(loss)/d(x).  1 / N = inv_n, or (DEV_COUNT: N over every rank) 1 / *count, read on the device.
template <bool ID, bool DEV_COUNT>
__global__ void __launch_bounds__(kEwThreads) repvgg_bwd_apply_kernel(const __nv_bfloat16* __restrict__ g, const __nv_bfloat16* __restrict__ a,
                                                                      const __nv_bfloat16* __restrict__ y3, const __nv_bfloat16* __restrict__ y1,
                                                                      const __nv_bfloat16* __restrict__ x, long long nvec, int C, RepvggStats st,
                                                                      const float* __restrict__ gamma3, const float* __restrict__ gamma1,
                                                                      const float* __restrict__ gamma_id, const float* __restrict__ sums, float inv_n,
                                                                      const double* __restrict__ count, __nv_bfloat16* __restrict__ dy3,
                                                                      __nv_bfloat16* __restrict__ dy1, __nv_bfloat16* __restrict__ dx_id) {
  if (DEV_COUNT) inv_n = (float)(1.0 / __ldg(count));
  const int cv = C / 8;
  for (long long i = blockIdx.x * (long long)kEwThreads + threadIdx.x; i < nvec; i += (long long)gridDim.x * kEwThreads) {
    const int c0 = (int)(i % cv) * 8;
    float fg[8], fa[8], f3[8], f1[8], fx[8];
    bf16x8_to_float(__ldg(reinterpret_cast<const uint4*>(g) + i), fg);
    bf16x8_to_float(__ldg(reinterpret_cast<const uint4*>(a) + i), fa);
    bf16x8_to_float(__ldg(reinterpret_cast<const uint4*>(y3) + i), f3);
    bf16x8_to_float(__ldg(reinterpret_cast<const uint4*>(y1) + i), f1);
    if (ID) bf16x8_to_float(__ldg(reinterpret_cast<const uint4*>(x) + i), fx);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int c = c0 + k;
      const float dz = fa[k] > 0.0f ? fg[k] : 0.0f;
      const float mdz = __ldg(sums + c) * inv_n;
      const float r3 = __ldg(st.s3 + C + c), r1 = __ldg(st.s1 + C + c);
      f3[k] = __ldg(gamma3 + c) * r3 * (dz - mdz - (f3[k] - __ldg(st.s3 + c)) * r3 * __ldg(sums + C + c) * inv_n);
      f1[k] = __ldg(gamma1 + c) * r1 * (dz - mdz - (f1[k] - __ldg(st.s1 + c)) * r1 * __ldg(sums + 2 * C + c) * inv_n);
      if (ID) {
        const float ri = __ldg(st.sid + C + c);
        fx[k] = __ldg(gamma_id + c) * ri * (dz - mdz - (fx[k] - __ldg(st.sid + c)) * ri * __ldg(sums + 3 * C + c) * inv_n);
      }
    }
    reinterpret_cast<uint4*>(dy3)[i] = float_to_bf16x8(f3);
    reinterpret_cast<uint4*>(dy1)[i] = float_to_bf16x8(f1);
    if (ID) reinterpret_cast<uint4*>(dx_id)[i] = float_to_bf16x8(fx);
  }
}

// BiFusion's ConvTranspose2d(c, c, 2, stride=2, bias) (src/models/modules/yolo_modules.py:245-265) around a 1x1 GEMM u [B,h,w,4c] whose
// column (py * 2 + px) * c + o is output pixel (2y + py, 2x + px), channel o.  Scatter: out [B,2h,2w,c] = u + bias (fp32 sum, one bf16
// rounding).  Item = one 8-channel vector of out.
__global__ void __launch_bounds__(kEwThreads) convt_scatter_kernel(const __nv_bfloat16* __restrict__ u, int B, int h, int w, int C,
                                                                   const float* __restrict__ bias, __nv_bfloat16* __restrict__ out) {
  const int cv = C / 8, W2 = 2 * w;
  const long long n = (long long)B * 4 * h * w * cv;
  for (long long i = blockIdx.x * (long long)kEwThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kEwThreads) {
    const int v = (int)(i % cv);
    const long long p = i / cv;
    const int X = (int)(p % W2);
    const long long t = p / W2;
    const int Y = (int)(t % (2 * h));
    const long long img = t / (2 * h);
    const long long src = ((img * h + Y / 2) * w + X / 2) * 4 * cv + ((Y & 1) * 2 + (X & 1)) * cv + v;
    float f[8];
    bf16x8_to_float(__ldg(reinterpret_cast<const uint4*>(u) + src), f);
#pragma unroll
    for (int k = 0; k < 8; ++k) f[k] += __ldg(bias + 8 * v + k);
    reinterpret_cast<uint4*>(out)[i] = float_to_bf16x8(f);
  }
}

// Gather: g = d(loss)/d(out) [B,2h,2w,c] -> du [B,h,w,4c] in the GEMM layout (a permutation: exact), and dbias partials: CTA b sums its
// fixed pixel range of g per channel (pixel lanes in order, then a fixed shared-memory tree over the lanes) into partial[b][c].
// convt_bias_finish_kernel adds the kConvtParts partials in order: dbias is bitwise reproducible.
constexpr int kConvtParts = 256;

__global__ void __launch_bounds__(kEwThreads) convt_gather_kernel(const __nv_bfloat16* __restrict__ g, int B, int h, int w, int C,
                                                                  __nv_bfloat16* __restrict__ du, float* __restrict__ partial) {
  __shared__ float s_part[kEwThreads * 8];
  const int cv = C / 8, W2 = 2 * w;
  const int v = threadIdx.x % cv;
  const int pl = threadIdx.x / cv, np = kEwThreads / cv;
  const bool active = pl < np;
  const long long npix = (long long)B * 4 * h * w;
  const long long chunk = (npix + gridDim.x - 1) / gridDim.x;
  const long long p0 = (long long)blockIdx.x * chunk, p1 = min(npix, p0 + chunk);
  float acc[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) acc[k] = 0.0f;
  if (active) {
    for (long long p = p0 + pl; p < p1; p += np) {
      const int X = (int)(p % W2);
      const long long t = p / W2;
      const int Y = (int)(t % (2 * h));
      const long long img = t / (2 * h);
      const uint4 q = __ldg(reinterpret_cast<const uint4*>(g) + p * cv + v);
      reinterpret_cast<uint4*>(du)[((img * h + Y / 2) * w + X / 2) * 4 * cv + ((Y & 1) * 2 + (X & 1)) * cv + v] = q;
      float f[8];
      bf16x8_to_float(q, f);
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[k] += f[k];
    }
  }
  // fixed tree over the pixel lanes: lane pl takes lane pl + s for s = the largest power of two below np, then halving
  if (active) {
#pragma unroll
    for (int k = 0; k < 8; ++k) s_part[pl * C + v * 8 + k] = acc[k];
  }
  __syncthreads();
  int s0 = 1;
  while (2 * s0 < np) s0 *= 2;
  for (int s = s0; s > 0; s >>= 1) {
    if (pl < s && pl + s < np) {
#pragma unroll
      for (int k = 0; k < 8; ++k) s_part[pl * C + v * 8 + k] += s_part[(pl + s) * C + v * 8 + k];
    }
    __syncthreads();
  }
  for (int c = threadIdx.x; c < C; c += kEwThreads) partial[(long long)blockIdx.x * C + c] = s_part[c];
}

__global__ void convt_bias_finish_kernel(const float* __restrict__ partial, int C, float* __restrict__ dbias) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float t = 0.0f;
  for (int b = 0; b < kConvtParts; ++b) t += partial[(long long)b * C + c];
  dbias[c] = t;
}

// fp32 master weights [cout][cin][kh][kw] (nn.Conv2d) -> bf16 [cout][kh*kw][cin] (forward / wgrad layout) and the backward-data operand
// bf16 [cin][kh*kw][cout] with the taps rotated by 180 degrees.  The K rows are kin_pad = kpad(cin) / kout_pad = kpad(cout) long (16 and 32
// channels: one zero-padded 64-channel chunk; the padding is zeroed by the caller)
__global__ void pack_train_weights_kernel(const float* __restrict__ w, int cout, int cin, int taps, int kin_pad, int kout_pad, __nv_bfloat16* __restrict__ wf,
                                          __nv_bfloat16* __restrict__ wb) {
  const long long n = (long long)cout * cin * taps;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int t = (int)(i % taps);
    const int ci = (int)((i / taps) % cin);
    const int co = (int)(i / ((long long)taps * cin));
    const __nv_bfloat16 v = __float2bfloat16_rn(w[i]);
    wf[((size_t)co * taps + t) * kin_pad + ci] = v;
    wb[((size_t)ci * taps + (taps - 1 - t)) * kout_pad + co] = v;
  }
}

// ------------------------------------------------------------------------------------------------ host
// every training operand is bf16 with 64-element (128-byte) K rows
static int encode_tiled(CUtensorMap* m, int rank, const void* base, const cuuint64_t* dims, const cuuint64_t* strides_bytes, const cuuint32_t* box) {
  return encode_map(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, base, dims, strides_bytes, box, CU_TENSOR_MAP_SWIZZLE_128B);
}

// pixel box TW x TH x NB with exactly 128 pixels (powers of two) that wastes the fewest rows on out-of-bounds pixels
static void choose_box128(int B, int H, int W, int* TW, int* TH, int* NB) {
  double best = -1.0;
  for (int tw = 1; tw <= 128; tw *= 2)
    for (int th = 1; tw * th <= 128; th *= 2) {
      const int nb = 128 / (tw * th);
      const double tiles = (double)ceil_div(W, tw) * ceil_div(H, th) * ceil_div(B, nb);
      const double util = (double)B * H * W / (tiles * 128.0) + 1e-6 * tw;
      if (util > best) {
        best = util;
        *TW = tw;
        *TH = th;
        *NB = nb;
      }
    }
}

static int act_map(CUtensorMap* m, const void* base, int B, int H, int W, int C, int TW, int TH, int NB) {
  const cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
  const cuuint64_t str[3] = {(cuuint64_t)C * 2, (cuuint64_t)C * 2 * W, (cuuint64_t)C * 2 * W * H};
  const cuuint32_t box[4] = {64, (cuuint32_t)TW, (cuuint32_t)TH, (cuuint32_t)NB};
  return encode_tiled(m, 4, base, dims, str, box);
}

}  // namespace cvb

using namespace cvb;

// channel counts of the training convolutions: 16, 32 (one partial K chunk / N tile) or multiples of 64
static bool train_channels_ok(int c) { return c == 16 || c == 32 || (c > 0 && c % 64 == 0); }
static int kpad64(int c) { return (c + 63) / 64 * 64; }

extern "C" int cvb_train_pack_weights(const float* w, int32_t cout, int32_t cin, int32_t k, void* w_fwd, void* w_bwd, void* stream) {
  CVB_REQUIRE(w && w_fwd && w_bwd && cout > 0 && cin > 0 && (k == 1 || k == 3), "train_pack_weights: bad argument");
  CVB_REQUIRE(train_channels_ok(cin) && train_channels_ok(cout), "train_pack_weights: channels must be 16, 32 or multiples of 64 (cin=%d cout=%d)", cin, cout);
  const long long n = (long long)cout * cin * k * k;
  const int kin = kpad64(cin), kout = kpad64(cout);
  cudaStream_t st = as_stream(stream);
  if (kin != cin) CVB_CHECK_CUDA(cudaMemsetAsync(w_fwd, 0, (size_t)cout * k * k * kin * 2, st));
  if (kout != cout) CVB_CHECK_CUDA(cudaMemsetAsync(w_bwd, 0, (size_t)cin * k * k * kout * 2, st));
  pack_train_weights_kernel<<<(int)((n + 255) / 256 < 1184 ? (n + 255) / 256 : 1184), 256, 0, st>>>(
      w, cout, cin, k * k, kin, kout, static_cast<__nv_bfloat16*>(w_fwd), static_cast<__nv_bfloat16*>(w_bwd));
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}

// m[py * 2 + px]: tensor map of the parity class (py, px) of an NHWC tensor, pixels (2i + py, 2j + px), the inputs of s2_taps' tap_map
static int parity_maps(CUtensorMap* m, const void* base, int B, int H, int W, int C, int TW, int TH, int NB) {
  const cuuint32_t box[4] = {64, (cuuint32_t)TW, (cuuint32_t)TH, (cuuint32_t)NB};
  int rc = CVB_OK;
  for (int p = 0; p < 4 && rc == CVB_OK; ++p) {
    const int py = p >> 1, px = p & 1;
    const int Wp = (W - px + 1) / 2, Hp = (H - py + 1) / 2;
    const cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)Wp, (cuuint64_t)Hp, (cuuint64_t)B};
    const cuuint64_t str[3] = {(cuuint64_t)C * 2 * 2, (cuuint64_t)C * 2 * W * 2, (cuuint64_t)C * 2 * W * H};
    if (Wp <= 0 || Hp <= 0) rc = act_map(&m[p], base, B, H, W, C, TW, TH, NB);  // no pixel of this parity, no tap reads it (s2_taps): any valid map
    else rc = encode_tiled(&m[p], 4, static_cast<const uint8_t*>(base) + ((size_t)py * W + px) * C * 2, dims, str, box);
  }
  return rc;
}

// stride 1, padding pad: tap t reads input pixel (h + t / k - pad, w + t % k - pad) of the one input map and weight K block t.  -> k * k
static int s1_taps(int k, int pad, int8_t* dh, int8_t* dw, int8_t* map, int8_t* tap) {
  for (int t = 0; t < k * k; ++t) {
    dh[t] = (int8_t)(t / k - pad);
    dw[t] = (int8_t)(t % k - pad);
    map[t] = 0;
    tap[t] = (int8_t)t;
  }
  return k * k;
}

// stride-2 3x3 / pad 1: tap (ky, kx) reads input pixel (2h + ky - 1, 2w + kx - 1) = parity class ((ky + 1) & 1, (kx + 1) & 1) at index
// (h + (ky == 0 ? -1 : 0), w + (kx == 0 ? -1 : 0)) of that class.  When H or W is 1 the odd class has no pixel: its taps read only padding
// and are left out.  -> number of taps kept; tap[i] = ky * 3 + kx of kept tap i
static int s2_taps(int H, int W, int8_t* dh, int8_t* dw, int8_t* map, int8_t* tap) {
  int n = 0;
  for (int ky = 0; ky < 3; ++ky)
    for (int kx = 0; kx < 3; ++kx) {
      const int py = (ky + 1) & 1, px = (kx + 1) & 1;
      if (H - py <= 0 || W - px <= 0) continue;
      dh[n] = (int8_t)(ky == 0 ? -1 : 0);
      dw[n] = (int8_t)(kx == 0 ? -1 : 0);
      map[n] = (int8_t)((py << 1) | px);
      tap[n] = (int8_t)(ky * 3 + kx);
      ++n;
    }
  return n;
}

// Zeroed launch arguments for an H x W x B tile grid whose point (h, w) writes pixel (h * os + ooh, w * os + oow) of the out_H x out_W
// tensor `out`, with the grid's 128-pixel box and tile counts.  The caller adds the taps and their input maps.
static void tconv_geometry(TConvArgs& a, int B, int H, int W, int cin, int cout, void* out, int out_H, int out_W, int os, int ooh, int oow) {
  memset(&a, 0, sizeof(a));
  a.B = B;
  a.H = H;
  a.W = W;
  a.cin = cin;
  a.cout = cout;
  a.out = static_cast<__nv_bfloat16*>(out);
  a.out_H = out_H;
  a.out_W = out_W;
  a.os = os;
  a.ooh = ooh;
  a.oow = oow;
  choose_box128(B, H, W, &a.TW, &a.TH, &a.NB);
  a.tiles_w = ceil_div(W, a.TW);
  a.tiles_h = ceil_div(H, a.TH);
  a.tiles_b = ceil_div(B, a.NB);
}

static int launch_tconv(TConvArgs& a, const void* w_packed, int wblocks, const void* y_prev, const float* bn_stat_prev, void* stream) {
  a.y_prev = static_cast<const __nv_bfloat16*>(y_prev);
  a.s_prev = bn_stat_prev ? bn_stat_prev + 2 * (size_t)a.cout : nullptr;
  a.t_prev = bn_stat_prev ? bn_stat_prev + 3 * (size_t)a.cout : nullptr;
  const int bn = a.cout % 128 == 0 ? 128 : (a.cout % 64 == 0 ? 64 : 32);  // 32: cout = 16 or 32, one tile (rows past cout zero-filled)
  {
    const long long K = (long long)wblocks * kpad64(a.cin);
    const cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)a.cout};
    const cuuint64_t str[1] = {(cuuint64_t)K * 2};
    const cuuint32_t box[2] = {64, (cuuint32_t)bn};
    const int rc = encode_tiled(&a.tmB, 2, w_packed, dims, str, box);
    if (rc != CVB_OK) return rc;
  }
  // tconv_kernel<BN, SILU_BWD, PRED> by [BN = 32, 64, 128][plain, SiLU' epilogue, PRED]
  const void* const fns[3][3] = {
      {reinterpret_cast<const void*>(&tconv_kernel<32, false>), reinterpret_cast<const void*>(&tconv_kernel<32, true>), reinterpret_cast<const void*>(&tconv_kernel<32, false, true>)},
      {reinterpret_cast<const void*>(&tconv_kernel<64, false>), reinterpret_cast<const void*>(&tconv_kernel<64, true>), reinterpret_cast<const void*>(&tconv_kernel<64, false, true>)},
      {reinterpret_cast<const void*>(&tconv_kernel<128, false>), reinterpret_cast<const void*>(&tconv_kernel<128, true>), reinterpret_cast<const void*>(&tconv_kernel<128, false, true>)}};
  const void* fn = fns[bn / 64][a.out_f32 ? 2 : (y_prev ? 1 : 0)];
  const int k_iters = a.taps * (kpad64(a.cin) / 64);
  a.stages = k_iters < kTStagesFwd ? k_iters : kTStagesFwd;
  const int smem = a.stages * (128 * 128 + bn * 128) + 256 + 2 * bn * 4;
  CVB_CHECK_CUDA(opt_in_smem(fn, smem));
  void* kargs[1] = {&a};
  const dim3 grid((unsigned)(a.tiles_w * a.tiles_h * a.tiles_b), (unsigned)ceil_div(a.cout, bn));
  CVB_CHECK_CUDA(cudaLaunchKernel(fn, grid, dim3(kTThreads), kargs, (size_t)smem, as_stream(stream)));
  count_launch();
  return CVB_OK;
}

// paddings of the stride-1 training convolutions: k // 2 (BaseConv), 1 on a 1x1 conv (the YOLOX head stems, heads/yolox_head.py:35) and
// k - 1 - 1 = -1, the backward-data of that stem
static bool train_pad_ok(int k, int pad) { return k == 1 ? (pad >= -1 && pad <= 1) : (k == 3 && pad == 1); }

// Shape rules of a training convolution (forward / backward-data and backward-weight alike).  a, b, c: the operands, which must be 16-byte
// aligned (c may be null).  A stride-1 output is (H + 2 pad - k + 1) x (W + 2 pad - k + 1): TMA zero-fills the pixels outside the input
// (pad > 0), a negative pad crops its border instead.
static int check_conv_shape(const char* fn, int B, int H, int W, int cin, int cout, int k, int stride, int pad, const void* a, const void* b,
                            const void* c = nullptr) {
  CVB_REQUIRE((k == 1 || k == 3) && train_channels_ok(cin) && train_channels_ok(cout),
              "%s: k in {1,3}, channels must be 16, 32 or multiples of 64 (cin=%d cout=%d k=%d)", fn, cin, cout, k);
  CVB_REQUIRE(stride == 1 || (stride == 2 && k == 3), "%s: stride 1, or stride 2 with k = 3", fn);
  CVB_REQUIRE(train_pad_ok(k, pad), "%s: padding must be -1, 0 or 1 with k = 1, and 1 with k = 3 (k=%d pad=%d)", fn, k, pad);
  CVB_REQUIRE(B > 0 && H > 0 && W > 0 && H + 2 * pad - k + 1 > 0 && W + 2 * pad - k + 1 > 0, "%s: empty output (B=%d H=%d W=%d k=%d pad=%d)", fn, B, H, W,
              k, pad);
  CVB_REQUIRE(is_aligned(a, 16) && is_aligned(b, 16) && is_aligned(c, 16), "%s: pointers must be 16-byte aligned", fn);
  return CVB_OK;
}

static int train_conv(const void* x, int B, int H, int W, int cin, const void* w_packed, int cout, int k, int stride, int pad, void* out, const void* y_prev,
                      const float* bn_stat_prev, void* stream) {
  CVB_REQUIRE(x && w_packed && out, "train_conv: null tensor");
  int rc = check_conv_shape("train_conv", B, H, W, cin, cout, k, stride, pad, x, w_packed, out);
  if (rc != CVB_OK) return rc;
  CVB_REQUIRE((y_prev == nullptr) == (bn_stat_prev == nullptr), "train_conv: the SiLU' epilogue needs both y_prev and its BN statistics");
  TConvArgs a;
  const int Ho = (H + 2 * pad - k) / stride + 1, Wo = (W + 2 * pad - k) / stride + 1;
  tconv_geometry(a, B, Ho, Wo, cin, cout, out, Ho, Wo, 1, 0, 0);
  if (stride == 1) {
    a.taps = s1_taps(k, pad, a.tap_dh, a.tap_dw, a.tap_map, a.tap_wblk);
    rc = act_map(&a.tmA[0], x, B, H, W, cin, a.TW, a.TH, a.NB);
  } else {
    a.taps = s2_taps(H, W, a.tap_dh, a.tap_dw, a.tap_map, a.tap_wblk);
    rc = parity_maps(a.tmA, x, B, H, W, cin, a.TW, a.TH, a.NB);
  }
  if (rc != CVB_OK) return rc;
  return launch_tconv(a, w_packed, k * k, y_prev, bn_stat_prev, stream);
}

extern "C" int cvb_train_conv(const void* x, int32_t B, int32_t H, int32_t W, int32_t cin, const void* w_packed, int32_t cout, int32_t k, int32_t stride, void* out,
                              const void* y_prev, const float* bn_stat_prev, void* stream) {
  return train_conv(x, B, H, W, cin, w_packed, cout, k, stride, k / 2, out, y_prev, bn_stat_prev, stream);
}

extern "C" int cvb_train_conv_pad(const void* x, int32_t B, int32_t H, int32_t W, int32_t cin, const void* w_packed, int32_t cout, int32_t k, int32_t pad, void* out,
                                  const void* y_prev, const float* bn_stat_prev, void* stream) {
  return train_conv(x, B, H, W, cin, w_packed, cout, k, 1, pad, out, y_prev, bn_stat_prev, stream);
}

// training width of a prediction conv's GEMM: the channels rounded up to 16, 32 or a multiple of 64
static int pred_cout_pad(int c) { return c <= 16 ? 16 : (c <= 32 ? 32 : kpad64(c)); }

extern "C" int cvb_train_pred_conv(const void* x, int32_t B, int32_t H, int32_t W, int32_t cin, const void* w_packed, int32_t cout, int32_t cout_pad,
                                   const float* bias, float* out, int32_t c_tot, int32_t c_off, void* stream) {
  CVB_REQUIRE(x && w_packed && bias && out, "train_pred_conv: null tensor");
  CVB_REQUIRE(train_channels_ok(cin) && B > 0 && H > 0 && W > 0, "train_pred_conv: cin must be 16, 32 or a multiple of 64 (cin=%d)", cin);
  CVB_REQUIRE(cout > 0 && cout_pad == pred_cout_pad(cout), "train_pred_conv: cout_pad must be the next training width of cout (cout=%d cout_pad=%d)", cout, cout_pad);
  CVB_REQUIRE(c_off >= 0 && c_off + cout <= c_tot, "train_pred_conv: channels [%d, %d) outside the %d-channel output", c_off, c_off + cout, c_tot);
  CVB_REQUIRE(is_aligned(x, 16) && is_aligned(w_packed, 16) && is_aligned(out, 4) && is_aligned(bias, 4),
              "train_pred_conv: x / w_packed must be 16-byte, out / bias 4-byte aligned");
  TConvArgs a;
  tconv_geometry(a, B, H, W, cin, cout_pad, nullptr, H, W, 1, 0, 0);
  a.taps = s1_taps(1, 0, a.tap_dh, a.tap_dw, a.tap_map, a.tap_wblk);
  const int rc = act_map(&a.tmA[0], x, B, H, W, cin, a.TW, a.TH, a.NB);
  if (rc != CVB_OK) return rc;
  a.out_f32 = out;
  a.bias = bias;
  a.c_tot = c_tot;
  a.c_off = c_off;
  a.n_store = cout;
  return launch_tconv(a, w_packed, 1, nullptr, nullptr, stream);
}

// Backward-data of the 3x3 / stride 2 / pad 1 convolution: dx[2a + pi, 2b + pj] gets dy[a + dh, b + dw] through the taps whose parity matches
// (pi = 0: ky = 1; pi = 1: ky = 0 (dh = +1) and ky = 2 (dh = 0); same for columns) -- four dense stride-1 sub-convolutions over dy, one per
// parity class of dx, each writing its class with a strided store.  w_bwd = the [cin][9][cout] operand of cvb_train_pack_weights (taps rotated).
extern "C" int cvb_train_conv_dgrad_s2(const void* dy, int32_t B, int32_t Ho, int32_t Wo, int32_t cout, const void* w_bwd, int32_t cin, int32_t H, int32_t W, void* dx,
                                       const void* y_prev, const float* bn_stat_prev, void* stream) {
  CVB_REQUIRE(dy && w_bwd && dx, "train_conv_dgrad_s2: null tensor");
  CVB_REQUIRE(train_channels_ok(cin) && train_channels_ok(cout), "train_conv_dgrad_s2: channels must be 16, 32 or multiples of 64 (cin=%d cout=%d)", cin, cout);
  CVB_REQUIRE(B > 0 && Ho == (H - 1) / 2 + 1 && Wo == (W - 1) / 2 + 1, "train_conv_dgrad_s2: bad geometry");
  CVB_REQUIRE((y_prev == nullptr) == (bn_stat_prev == nullptr), "train_conv_dgrad_s2: the SiLU' epilogue needs both y_prev and its BN statistics");
  for (int pi = 0; pi < 2; ++pi)
    for (int pj = 0; pj < 2; ++pj) {
      const int Hs = (H - pi + 1) / 2, Ws = (W - pj + 1) / 2;  // pixels of this parity class
      if (Hs <= 0 || Ws <= 0) continue;
      TConvArgs a;
      tconv_geometry(a, B, Hs, Ws, cout, cin, dx, H, W, 2, pi, pj);  // the GEMM's K: dy channels, its N: dx channels
      int nt = 0;
      for (int ky = 0; ky < 3; ++ky) {
        if (((ky + 1) & 1) != pi) continue;  // rows of parity pi are reached by ky with 2*oh + ky - 1 = ih
        for (int kx = 0; kx < 3; ++kx) {
          if (((kx + 1) & 1) != pj) continue;
          a.tap_dh[nt] = (int8_t)(ky == 0 ? 1 : 0);
          a.tap_dw[nt] = (int8_t)(kx == 0 ? 1 : 0);
          a.tap_map[nt] = 0;
          a.tap_wblk[nt] = (int8_t)(8 - (ky * 3 + kx));  // w_bwd stores tap t of the forward filter at block 8 - t
          ++nt;
        }
      }
      a.taps = nt;
      int rc = act_map(&a.tmA[0], dy, B, Ho, Wo, cout, a.TW, a.TH, a.NB);
      if (rc != CVB_OK) return rc;
      rc = launch_tconv(a, w_bwd, 9, y_prev, bn_stat_prev, stream);
      if (rc != CVB_OK) return rc;
    }
  return CVB_OK;
}

static int train_conv_wgrad(const void* x, const void* dy, int B, int H, int W, int cin, int cout, int k, int stride, int pad, float* dw, void* stream) {
  CVB_REQUIRE(x && dy && dw, "train_conv_wgrad: null tensor");
  int rc = check_conv_shape("train_conv_wgrad", B, H, W, cin, cout, k, stride, pad, x, dy);
  if (rc != CVB_OK) return rc;
  TWgradArgs a;
  memset(&a, 0, sizeof(a));
  const int Ho = (H + 2 * pad - k) / stride + 1, Wo = (W + 2 * pad - k) / stride + 1;
  choose_box128(B, Ho, Wo, &a.TW, &a.TH, &a.NB);
  a.tiles_w = ceil_div(Wo, a.TW);
  a.tiles_h = ceil_div(Ho, a.TH);
  a.tiles_b = ceil_div(B, a.NB);
  a.cin = cin;
  a.cout = cout;
  a.taps = k * k;
  a.dw = dw;
  const int m_tiles = a.tiles_w * a.tiles_h * a.tiles_b;
  const int cblocks = ceil_div(cin, 128);
  // widest block (4, 2 or 1 panels of 64) that divides cout: 192 runs as three 64-wide blocks, 384 as three 128-wide ones
  // (cout = 16 or 32: one 64-wide block whose columns past cout are not stored)
  const bool narrow = cout < 64;
  const int npan = narrow ? 1 : ((cout / 64) % 4 == 0 ? 4 : ((cout / 64) % 2 == 0 ? 2 : 1));
  a.nblocks = narrow ? 1 : cout / (64 * npan);
  const int sms = sm_count();
  if (sms == 0) return CVB_ERR_NO_DEVICE;
  int splits = (2 * sms) / (a.taps * cblocks * a.nblocks);  // ~two waves of CTAs: (split, tap, cin block x cout block)
  if (splits < 1) splits = 1;
  if (splits > m_tiles) splits = m_tiles;
  a.splits = splits;
  int ntaps;
  if (stride == 1) {
    ntaps = s1_taps(k, pad, a.tap_dh, a.tap_dw, a.tap_map, a.tap_idx);
    rc = act_map(&a.tmX[0], x, B, H, W, cin, a.TW, a.TH, a.NB);
  } else {
    ntaps = s2_taps(H, W, a.tap_dh, a.tap_dw, a.tap_map, a.tap_idx);  // the taps left out keep dw = 0
    rc = parity_maps(a.tmX, x, B, H, W, cin, a.TW, a.TH, a.NB);
  }
  if (rc == CVB_OK) rc = act_map(&a.tmD, dy, B, Ho, Wo, cout, a.TW, a.TH, a.NB);
  if (rc != CVB_OK) return rc;
  // twgrad_kernel<NPAN> for NPAN = 1, 2, 4 (index npan / 2); twgrad_kernel<1, true> for cout = 16 or 32
  const void* const fns[3] = {reinterpret_cast<const void*>(&twgrad_kernel<1>), reinterpret_cast<const void*>(&twgrad_kernel<2>),
                              reinterpret_cast<const void*>(&twgrad_kernel<4>)};
  const void* fn = narrow ? reinterpret_cast<const void*>(&twgrad_kernel<1, true>) : fns[npan / 2];
  const int stages = npan == 4 ? 2 : kTStagesWg;
  const int smem = stages * ((2 + npan) * 128 * 128) + 256;
  CVB_REQUIRE(smem <= 232448, "train_conv_wgrad: cout=%d needs %d bytes of shared memory", cout, smem);
  CVB_CHECK_CUDA(opt_in_smem(fn, smem));
  void* kargs[1] = {&a};
  const dim3 grid((unsigned)splits, (unsigned)ntaps, (unsigned)(cblocks * a.nblocks));
  CVB_CHECK_CUDA(cudaLaunchKernel(fn, grid, dim3(kTThreads), kargs, (size_t)smem, as_stream(stream)));
  count_launch();
  return CVB_OK;
}

extern "C" int cvb_train_conv_wgrad(const void* x, const void* dy, int32_t B, int32_t H, int32_t W, int32_t cin, int32_t cout, int32_t k, int32_t stride, float* dw,
                                    void* stream) {
  return train_conv_wgrad(x, dy, B, H, W, cin, cout, k, stride, k / 2, dw, stream);
}

extern "C" int cvb_train_conv_wgrad_pad(const void* x, const void* dy, int32_t B, int32_t H, int32_t W, int32_t cin, int32_t cout, int32_t k, int32_t pad, float* dw,
                                        void* stream) {
  return train_conv_wgrad(x, dy, B, H, W, cin, cout, k, 1, pad, dw, stream);
}

// Grids of the reduction and element-wise kernels; 0 when there is no device (sm_count() has set CVB_ERR_NO_DEVICE, which the caller
// returns).  Reduction kernels: `np` pixel lanes per CTA, at least ~4 pixels per thread, at most four CTAs per SM (2C global atomics per CTA).
static int red_grid(long long npix, int np) {
  long long g = (npix + (long long)np * 4 - 1) / ((long long)np * 4);
  const long long cap = (long long)sm_count() * 4;
  return (int)(cap == 0 ? 0 : g < 1 ? 1 : (g > cap ? cap : g));
}

static int ew_grid(long long work_items) {
  long long g = (work_items + kEwThreads - 1) / kEwThreads;
  const long long cap = (long long)sm_count() * 8;
  return (int)(cap == 0 ? 0 : g < 1 ? 1 : (g > cap ? cap : g));
}

// the npix / C rule of the SyncBatchNorm entry points (one lane per 8 channels of a kEwThreads-thread CTA)
static int check_bn_shape(const char* fn, int64_t npix, int32_t C) {
  CVB_REQUIRE(npix > 0 && C > 0 && C % 8 == 0 && C / 8 <= kEwThreads, "%s: npix must be > 0 and C a multiple of 8 up to 2048 (npix=%lld C=%d)", fn,
              (long long)npix, C);
  return CVB_OK;
}

extern "C" int cvb_train_bn_stats(const void* y, int64_t npix, int32_t C, const float* gamma, const float* beta, float eps, float momentum, float* running_mean,
                                  float* running_var, float* sums_scratch, float* stat, void* stream) {
  CVB_REQUIRE(y && gamma && beta && sums_scratch && stat && npix > 0 && C % 8 == 0 && C <= 2048, "train_bn_stats: bad argument");
  cudaStream_t st = as_stream(stream);
  CVB_CHECK_CUDA(cudaMemsetAsync(sums_scratch, 0, 2 * (size_t)C * sizeof(float), st));
  const int np = kEwThreads / (C / 8) > 0 ? kEwThreads / (C / 8) : 1;
  CVB_REQUIRE(C / 8 <= kEwThreads, "train_bn_stats: C too large");
  const int grid = red_grid(npix, np);
  if (grid == 0) return CVB_ERR_NO_DEVICE;
  bn_stats_kernel<<<grid, kEwThreads, 0, st>>>(static_cast<const __nv_bfloat16*>(y), npix, C, sums_scratch);
  bn_finalize_kernel<<<ceil_div(C, 128), 128, 0, st>>>(sums_scratch, static_cast<const __nv_bfloat16*>(y), npix, C, gamma, beta, eps, momentum, running_mean, running_var, stat);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch(2);
  return CVB_OK;
}

template <int ACT>
static int bn_act_fwd(const void* y, int64_t npix, int32_t C, const float* stat, void* out, void* stream) {
  const long long nvec = npix * (C / 8);
  const int grid = ew_grid(nvec);
  if (grid == 0) return CVB_ERR_NO_DEVICE;
  bn_act_fwd_kernel<ACT><<<grid, kEwThreads, 0, as_stream(stream)>>>(static_cast<const __nv_bfloat16*>(y), nvec, C, stat, static_cast<__nv_bfloat16*>(out));
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}

extern "C" int cvb_train_bn_silu_fwd(const void* y, int64_t npix, int32_t C, const float* stat, void* out, void* stream) {
  CVB_REQUIRE(y && stat && out && C % 8 == 0, "train_bn_silu_fwd: bad argument");
  return bn_act_fwd<kActSilu>(y, npix, C, stat, out, stream);
}

template <int ACT = kActSilu>
static int bn_bwd_reduce(const void* g, int32_t g_is_dz, const void* y, int64_t npix, int32_t C, const float* stat, float* sums, cudaStream_t st) {
  CVB_CHECK_CUDA(cudaMemsetAsync(sums, 0, 2 * (size_t)C * sizeof(float), st));
  const int grid = red_grid(npix, kEwThreads / (C / 8));
  if (grid == 0) return CVB_ERR_NO_DEVICE;
  bn_act_bwd_reduce_kernel<ACT><<<grid, kEwThreads, 0, st>>>(
      static_cast<const __nv_bfloat16*>(g), static_cast<const __nv_bfloat16*>(y), npix, C, stat, g_is_dz, sums);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}

// count == nullptr: 1 / npix (this device's pixels); otherwise 1 / *count, the global count bn_merge_kernel left on the device
template <int ACT = kActSilu>
static int bn_bwd_apply(const void* g, int32_t g_is_dz, const void* y, int64_t npix, int32_t C, const float* stat, const float* gamma, const float* sums,
                        const double* count, void* dy, cudaStream_t st) {
  const long long nvec = npix * (C / 8);
  const int grid = ew_grid(nvec);
  if (grid == 0) return CVB_ERR_NO_DEVICE;
  const auto* gb = static_cast<const __nv_bfloat16*>(g);
  const auto* yb = static_cast<const __nv_bfloat16*>(y);
  auto* dyb = static_cast<__nv_bfloat16*>(dy);
  if (count == nullptr)
    bn_act_bwd_apply_kernel<ACT, false><<<grid, kEwThreads, 0, st>>>(gb, yb, nvec, C, stat, gamma, sums, (float)(1.0 / (double)npix), nullptr, g_is_dz, dyb);
  else
    bn_act_bwd_apply_kernel<ACT, true><<<grid, kEwThreads, 0, st>>>(gb, yb, nvec, C, stat, gamma, sums, 0.0f, count, g_is_dz, dyb);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}

extern "C" int cvb_train_bn_silu_bwd(const void* g, int32_t g_is_dz, const void* y, int64_t npix, int32_t C, const float* stat, const float* gamma, float* sums /* [2][C]: out = dbeta, dgamma */,
                                     void* dy, void* stream) {
  CVB_REQUIRE(g && y && stat && gamma && sums && dy && C % 8 == 0 && C / 8 <= kEwThreads, "train_bn_silu_bwd: bad argument");
  cudaStream_t st = as_stream(stream);
  const int rc = bn_bwd_reduce(g, g_is_dz, y, npix, C, stat, sums, st);
  return rc != CVB_OK ? rc : bn_bwd_apply(g, g_is_dz, y, npix, C, stat, gamma, sums, nullptr, dy, st);
}

// ---- SyncBatchNorm: the statistics and the backward split where a collective sits between the two halves
extern "C" int cvb_train_bn_partial(const void* y, int64_t npix, int32_t C, float* sums_scratch, double* record, void* stream) {
  CVB_REQUIRE(y && sums_scratch && record, "train_bn_partial: null pointer");
  const int rc = check_bn_shape("train_bn_partial", npix, C);
  if (rc != CVB_OK) return rc;
  CVB_REQUIRE(is_aligned(y, 16) && is_aligned(record, 8), "train_bn_partial: y must be 16-byte, record 8-byte aligned");
  cudaStream_t st = as_stream(stream);
  CVB_CHECK_CUDA(cudaMemsetAsync(sums_scratch, 0, 2 * (size_t)C * sizeof(float), st));
  const int grid = red_grid(npix, kEwThreads / (C / 8));
  if (grid == 0) return CVB_ERR_NO_DEVICE;
  bn_stats_kernel<<<grid, kEwThreads, 0, st>>>(static_cast<const __nv_bfloat16*>(y), npix, C, sums_scratch);
  bn_partial_kernel<<<ceil_div(C, 128), 128, 0, st>>>(sums_scratch, static_cast<const __nv_bfloat16*>(y), npix, C, record);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch(2);
  return CVB_OK;
}

extern "C" int cvb_train_bn_merge(const double* records, int32_t world, int32_t C, const float* gamma, const float* beta, float eps, float momentum,
                                  float* running_mean, float* running_var, float* stat, double* count, void* stream) {
  CVB_REQUIRE(records && gamma && beta && stat && count, "train_bn_merge: null pointer");
  CVB_REQUIRE((running_mean == nullptr) == (running_var == nullptr), "train_bn_merge: running_mean and running_var go together");
  CVB_REQUIRE(world >= 1 && C > 0 && C % 8 == 0 && C <= 2048, "train_bn_merge: world must be >= 1 and C a multiple of 8 up to 2048 (world=%d C=%d)", world, C);
  CVB_REQUIRE(is_aligned(records, 8) && is_aligned(count, 8), "train_bn_merge: records / count must be 8-byte aligned");
  bn_merge_kernel<<<ceil_div(C, 128), 128, 0, as_stream(stream)>>>(records, world, C, gamma, beta, eps, momentum, running_mean, running_var, stat, count);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}

extern "C" int cvb_train_bn_silu_bwd_reduce(const void* g, int32_t g_is_dz, const void* y, int64_t npix, int32_t C, const float* stat, float* sums, void* stream) {
  CVB_REQUIRE(g && y && stat && sums, "train_bn_silu_bwd_reduce: null pointer");
  const int rc = check_bn_shape("train_bn_silu_bwd_reduce", npix, C);
  return rc != CVB_OK ? rc : bn_bwd_reduce(g, g_is_dz, y, npix, C, stat, sums, as_stream(stream));
}

extern "C" int cvb_train_bn_silu_bwd_apply(const void* g, int32_t g_is_dz, const void* y, int64_t npix, int32_t C, const float* stat, const float* gamma,
                                           const float* sums, const double* count, void* dy, void* stream) {
  CVB_REQUIRE(g && y && stat && gamma && sums && count && dy, "train_bn_silu_bwd_apply: null pointer");
  const int rc = check_bn_shape("train_bn_silu_bwd_apply", npix, C);
  if (rc != CVB_OK) return rc;
  CVB_REQUIRE(is_aligned(count, 8), "train_bn_silu_bwd_apply: count must be 8-byte aligned");
  return bn_bwd_apply(g, g_is_dz, y, npix, C, stat, gamma, sums, count, dy, as_stream(stream));
}

extern "C" int cvb_train_focus_s2d(const float* img, int32_t B, int32_t H, int32_t W, void* out, void* stream) {
  CVB_REQUIRE(img && out && B > 0 && H > 0 && W > 0, "train_focus_s2d: bad argument");
  CVB_REQUIRE(H % 2 == 0 && W % 2 == 0, "train_focus_s2d: H and W must be even (H=%d W=%d)", H, W);
  CVB_REQUIRE(is_aligned(img, 8) && is_aligned(out, 16), "train_focus_s2d: img must be 8-byte, out 16-byte aligned");
  const int grid = ew_grid((long long)B * (H / 2) * (W / 2));
  if (grid == 0) return CVB_ERR_NO_DEVICE;
  focus_s2d_kernel<<<grid, kEwThreads, 0, as_stream(stream)>>>(img, B, H, W, static_cast<__nv_bfloat16*>(out));
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}

extern "C" int cvb_train_spp_pool_fwd(const void* a, int32_t B, int32_t H, int32_t W, int32_t C, void* cat, void* idx, void* stream) {
  CVB_REQUIRE(a && cat && idx && B > 0 && H > 0 && W > 0 && C > 0, "train_spp_pool_fwd: bad argument");
  CVB_REQUIRE(C % 8 == 0, "train_spp_pool_fwd: C must be a multiple of 8 (C=%d)", C);
  CVB_REQUIRE(is_aligned(a, 16) && is_aligned(cat, 16) && is_aligned(idx, 8), "train_spp_pool_fwd: a / cat must be 16-byte, idx 8-byte aligned");
  const int grid = ew_grid((long long)B * H * W * (C / 8));
  if (grid == 0) return CVB_ERR_NO_DEVICE;
  spp_pool_fwd_kernel<<<grid, kEwThreads, 0, as_stream(stream)>>>(static_cast<const __nv_bfloat16*>(a), B, H, W, C, static_cast<__nv_bfloat16*>(cat),
                                                                         static_cast<uint8_t*>(idx));
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}

extern "C" int cvb_train_spp_pool_bwd(const void* g, const void* idx, int32_t B, int32_t H, int32_t W, int32_t C, void* da, void* stream) {
  CVB_REQUIRE(g && idx && da && B > 0 && H > 0 && W > 0 && C > 0, "train_spp_pool_bwd: bad argument");
  CVB_REQUIRE(C % 8 == 0, "train_spp_pool_bwd: C must be a multiple of 8 (C=%d)", C);
  CVB_REQUIRE(is_aligned(g, 16) && is_aligned(da, 16) && is_aligned(idx, 8), "train_spp_pool_bwd: g / da must be 16-byte, idx 8-byte aligned");
  const int grid = ew_grid((long long)B * H * W * (C / 8));
  if (grid == 0) return CVB_ERR_NO_DEVICE;
  spp_pool_bwd_kernel<<<grid, kEwThreads, 0, as_stream(stream)>>>(static_cast<const __nv_bfloat16*>(g), static_cast<const uint8_t*>(idx), B, H, W, C,
                                                                         static_cast<__nv_bfloat16*>(da));
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}

extern "C" int cvb_train_sppf_chain_fwd(const void* a, int32_t B, int32_t H, int32_t W, int32_t C, void* cat, void* idx, void* stream) {
  CVB_REQUIRE(a && cat && idx && B > 0 && H > 0 && W > 0 && C > 0, "train_sppf_chain_fwd: bad argument");
  CVB_REQUIRE(C % 8 == 0, "train_sppf_chain_fwd: C must be a multiple of 8 (C=%d)", C);
  CVB_REQUIRE(is_aligned(a, 16) && is_aligned(cat, 16), "train_sppf_chain_fwd: a / cat must be 16-byte aligned");
  cudaStream_t st = as_stream(stream);
  const long long n = (long long)B * H * W * C;
  const int pool_grid = ew_grid(n / 8), idx_grid = ew_grid(n);
  if (pool_grid == 0 || idx_grid == 0) return CVB_ERR_NO_DEVICE;
  spp_pool_fwd_kernel<<<pool_grid, kEwThreads, 0, st>>>(static_cast<const __nv_bfloat16*>(a), B, H, W, C, static_cast<__nv_bfloat16*>(cat), nullptr);
  sppf_chain_idx_kernel<<<idx_grid, kEwThreads, 0, st>>>(static_cast<const __nv_bfloat16*>(cat), B, H, W, C, static_cast<uint8_t*>(idx));
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch(2);
  return CVB_OK;
}

extern "C" int cvb_train_sppf_chain_bwd(const void* g, const void* idx, int32_t B, int32_t H, int32_t W, int32_t C, float* scratch, void* da, void* stream) {
  CVB_REQUIRE(g && idx && scratch && da && B > 0 && H > 0 && W > 0 && C > 0, "train_sppf_chain_bwd: bad argument");
  CVB_REQUIRE(is_aligned(g, 4) && is_aligned(da, 4) && is_aligned(scratch, 4), "train_sppf_chain_bwd: g / scratch / da must be 4-byte aligned");
  cudaStream_t st = as_stream(stream);
  const long long n = (long long)B * H * W * C;
  const int grid = ew_grid(n);
  if (grid == 0) return CVB_ERR_NO_DEVICE;
  const __nv_bfloat16* gb = static_cast<const __nv_bfloat16*>(g);
  const uint8_t* ib = static_cast<const uint8_t*>(idx);
  sppf_chain_bwd_kernel<<<grid, kEwThreads, 0, st>>>(gb, ib, 2, nullptr, scratch, nullptr, B, H, W, C);
  sppf_chain_bwd_kernel<<<grid, kEwThreads, 0, st>>>(gb, ib, 1, scratch, scratch + n, nullptr, B, H, W, C);
  sppf_chain_bwd_kernel<<<grid, kEwThreads, 0, st>>>(gb, ib, 0, scratch + n, nullptr, static_cast<__nv_bfloat16*>(da), B, H, W, C);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch(3);
  return CVB_OK;
}

extern "C" int cvb_train_upsample_cat_fwd(const void* a, int32_t B, int32_t h, int32_t w, int32_t Ca, const void* b, int32_t Cb, void* cat, void* stream) {
  CVB_REQUIRE(a && b && cat && B > 0 && h > 0 && w > 0 && Ca > 0 && Cb > 0, "train_upsample_cat_fwd: bad argument");
  CVB_REQUIRE(Ca % 8 == 0 && Cb % 8 == 0, "train_upsample_cat_fwd: channels must be multiples of 8 (Ca=%d Cb=%d)", Ca, Cb);
  CVB_REQUIRE(is_aligned(a, 16) && is_aligned(b, 16) && is_aligned(cat, 16), "train_upsample_cat_fwd: pointers must be 16-byte aligned");
  const int grid = ew_grid((long long)B * 4 * h * w * ((Ca + Cb) / 8));
  if (grid == 0) return CVB_ERR_NO_DEVICE;
  upsample_cat_fwd_kernel<<<grid, kEwThreads, 0, as_stream(stream)>>>(static_cast<const __nv_bfloat16*>(a), B, h, w, Ca, static_cast<const __nv_bfloat16*>(b),
                                                                             Cb, static_cast<__nv_bfloat16*>(cat));
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}

extern "C" int cvb_train_upsample_cat_bwd(const void* g, int32_t B, int32_t h, int32_t w, int32_t Ca, int32_t Cb, void* da, void* db, void* stream) {
  CVB_REQUIRE(g && da && db && B > 0 && h > 0 && w > 0 && Ca > 0 && Cb > 0, "train_upsample_cat_bwd: bad argument");
  CVB_REQUIRE(Ca % 8 == 0 && Cb % 8 == 0, "train_upsample_cat_bwd: channels must be multiples of 8 (Ca=%d Cb=%d)", Ca, Cb);
  CVB_REQUIRE(is_aligned(g, 16) && is_aligned(da, 16) && is_aligned(db, 16), "train_upsample_cat_bwd: pointers must be 16-byte aligned");
  const int grid = ew_grid((long long)B * h * w * (Ca / 8) + (long long)B * 4 * h * w * (Cb / 8));
  if (grid == 0) return CVB_ERR_NO_DEVICE;
  upsample_cat_bwd_kernel<<<grid, kEwThreads, 0, as_stream(stream)>>>(static_cast<const __nv_bfloat16*>(g), B, h, w, Ca, Cb, static_cast<__nv_bfloat16*>(da),
                                                                             static_cast<__nv_bfloat16*>(db));
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}

extern "C" int cvb_train_pred_grad(const float* g, int32_t B, int32_t c_tot, int32_t h, int32_t w, int32_t c_off, int32_t cout, int32_t cout_pad, void* dy, float* dbias,
                                   void* stream) {
  CVB_REQUIRE(g && dy && dbias && B > 0 && h > 0 && w > 0, "train_pred_grad: bad argument");
  CVB_REQUIRE(cout > 0 && cout_pad == pred_cout_pad(cout), "train_pred_grad: cout_pad must be the next training width of cout (cout=%d cout_pad=%d)", cout, cout_pad);
  CVB_REQUIRE(c_off >= 0 && c_off + cout <= c_tot, "train_pred_grad: channels [%d, %d) outside the %d-channel gradient", c_off, c_off + cout, c_tot);
  CVB_REQUIRE(is_aligned(dy, 16) && is_aligned(g, 4) && is_aligned(dbias, 4), "train_pred_grad: dy must be 16-byte, g / dbias 4-byte aligned");
  cudaStream_t st = as_stream(stream);
  const long long hw = (long long)h * w;
  const int grid = ew_grid((long long)B * hw * (cout_pad / 8));
  if (grid == 0) return CVB_ERR_NO_DEVICE;
  pred_grad_nhwc_kernel<<<grid, kEwThreads, 0, st>>>(g, B, c_tot, hw, c_off, cout, cout_pad, static_cast<__nv_bfloat16*>(dy));
  pred_bias_grad_kernel<<<cout, kEwThreads, 0, st>>>(g, B, c_tot, hw, c_off, dbias);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch(2);
  return CVB_OK;
}

// ---- YOLOv6: BatchNorm + ReLU, RepVGG branch sum, ConvTranspose2d scatter / gather
// every bf16 operand 16-byte aligned, C a multiple of 8 up to 2048 (one lane per 8 channels of a kEwThreads-thread CTA)
static bool aligned16(const void* p) { return p == nullptr || is_aligned(p, 16); }

extern "C" int cvb_train_bn_relu_fwd(const void* y, int64_t npix, int32_t C, const float* stat, void* out, void* stream) {
  CVB_REQUIRE(y && stat && out, "train_bn_relu_fwd: null pointer");
  const int rc = check_bn_shape("train_bn_relu_fwd", npix, C);
  if (rc != CVB_OK) return rc;
  CVB_REQUIRE(is_aligned(y, 16) && is_aligned(out, 16) && is_aligned(stat, 4), "train_bn_relu_fwd: y / out must be 16-byte, stat 4-byte aligned");
  return bn_act_fwd<kActRelu>(y, npix, C, stat, out, stream);
}

extern "C" int cvb_train_bn_relu_bwd(const void* g, const void* y, int64_t npix, int32_t C, const float* stat, const float* gamma, float* sums, void* dy,
                                     void* stream) {
  CVB_REQUIRE(g && y && stat && gamma && sums && dy, "train_bn_relu_bwd: null pointer");
  const int rc = check_bn_shape("train_bn_relu_bwd", npix, C);
  if (rc != CVB_OK) return rc;
  CVB_REQUIRE(is_aligned(g, 16) && is_aligned(y, 16) && is_aligned(dy, 16), "train_bn_relu_bwd: g / y / dy must be 16-byte aligned");
  CVB_REQUIRE(is_aligned(stat, 4) && is_aligned(gamma, 4) && is_aligned(sums, 4), "train_bn_relu_bwd: stat / gamma / sums must be 4-byte aligned");
  cudaStream_t st = as_stream(stream);
  const int r = bn_bwd_reduce<kActRelu>(g, 0, y, npix, C, stat, sums, st);
  return r != CVB_OK ? r : bn_bwd_apply<kActRelu>(g, 0, y, npix, C, stat, gamma, sums, nullptr, dy, st);
}

// SyncBatchNorm halves of cvb_train_bn_relu_bwd (a collective sums `sums` over the ranks between them)
extern "C" int cvb_train_bn_relu_bwd_reduce(const void* g, const void* y, int64_t npix, int32_t C, const float* stat, float* sums, void* stream) {
  CVB_REQUIRE(g && y && stat && sums, "train_bn_relu_bwd_reduce: null pointer");
  const int rc = check_bn_shape("train_bn_relu_bwd_reduce", npix, C);
  if (rc != CVB_OK) return rc;
  CVB_REQUIRE(is_aligned(g, 16) && is_aligned(y, 16), "train_bn_relu_bwd_reduce: g / y must be 16-byte aligned");
  CVB_REQUIRE(is_aligned(stat, 4) && is_aligned(sums, 4), "train_bn_relu_bwd_reduce: stat / sums must be 4-byte aligned");
  return bn_bwd_reduce<kActRelu>(g, 0, y, npix, C, stat, sums, as_stream(stream));
}

extern "C" int cvb_train_bn_relu_bwd_apply(const void* g, const void* y, int64_t npix, int32_t C, const float* stat, const float* gamma, const float* sums,
                                           const double* count, void* dy, void* stream) {
  CVB_REQUIRE(g && y && stat && gamma && sums && count && dy, "train_bn_relu_bwd_apply: null pointer");
  const int rc = check_bn_shape("train_bn_relu_bwd_apply", npix, C);
  if (rc != CVB_OK) return rc;
  CVB_REQUIRE(is_aligned(g, 16) && is_aligned(y, 16) && is_aligned(dy, 16), "train_bn_relu_bwd_apply: g / y / dy must be 16-byte aligned");
  CVB_REQUIRE(is_aligned(stat, 4) && is_aligned(gamma, 4) && is_aligned(sums, 4) && is_aligned(count, 8),
              "train_bn_relu_bwd_apply: stat / gamma / sums must be 4-byte, count 8-byte aligned");
  return bn_bwd_apply<kActRelu>(g, 0, y, npix, C, stat, gamma, sums, count, dy, as_stream(stream));
}

// the identity branch's operands come together: all of (x, stat_id[, gamma_id, dx_id]) or none
static int check_repvgg(const char* fn, int64_t npix, int32_t C, const void* x, const float* stat_id, const void* const* bf16s, int nb,
                        const float* const* f32s, int nf) {
  const int rc = check_bn_shape(fn, npix, C);
  if (rc != CVB_OK) return rc;
  for (int i = 0; i < nb; ++i) CVB_REQUIRE(aligned16(bf16s[i]), "%s: bf16 tensors must be 16-byte aligned", fn);
  for (int i = 0; i < nf; ++i) CVB_REQUIRE(f32s[i] == nullptr || is_aligned(f32s[i], 4), "%s: fp32 stat / gamma / sums must be 4-byte aligned", fn);
  CVB_REQUIRE((x == nullptr) == (stat_id == nullptr), "%s: x and stat_id go together (both NULL: no identity branch)", fn);
  return CVB_OK;
}

extern "C" int cvb_train_repvgg_fwd(const void* y3, const void* y1, const void* x, int64_t npix, int32_t C, const float* stat3, const float* stat1,
                                    const float* stat_id, void* out, void* stream) {
  CVB_REQUIRE(y3 && y1 && stat3 && stat1 && out, "train_repvgg_fwd: null pointer");
  const void* bf[] = {y3, y1, x, out};
  const float* f32[] = {stat3, stat1, stat_id};
  const int rc = check_repvgg("train_repvgg_fwd", npix, C, x, stat_id, bf, 4, f32, 3);
  if (rc != CVB_OK) return rc;
  const long long nvec = npix * (C / 8);
  const int grid = ew_grid(nvec);
  if (grid == 0) return CVB_ERR_NO_DEVICE;
  const RepvggStats st{stat3, stat1, stat_id};
  const auto* b3 = static_cast<const __nv_bfloat16*>(y3);
  const auto* b1 = static_cast<const __nv_bfloat16*>(y1);
  const auto* bx = static_cast<const __nv_bfloat16*>(x);
  auto* bo = static_cast<__nv_bfloat16*>(out);
  if (x)
    repvgg_fwd_kernel<true><<<grid, kEwThreads, 0, as_stream(stream)>>>(b3, b1, bx, nvec, C, st, bo);
  else
    repvgg_fwd_kernel<false><<<grid, kEwThreads, 0, as_stream(stream)>>>(b3, b1, nullptr, nvec, C, st, bo);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}

// The two halves of the RepVGG backward, shared by the fused entry and the SyncBatchNorm split.  Arguments checked by the caller.
static int repvgg_bwd_reduce(const void* g, const void* a, const void* y3, const void* y1, const void* x, int64_t npix, int32_t C, const RepvggStats& s,
                             float* sums, cudaStream_t st) {
  CVB_CHECK_CUDA(cudaMemsetAsync(sums, 0, 4 * (size_t)C * sizeof(float), st));
  const int grid = red_grid(npix, kEwThreads / (C / 8));
  if (grid == 0) return CVB_ERR_NO_DEVICE;
  const auto* bg = static_cast<const __nv_bfloat16*>(g);
  const auto* ba = static_cast<const __nv_bfloat16*>(a);
  const auto* b3 = static_cast<const __nv_bfloat16*>(y3);
  const auto* b1 = static_cast<const __nv_bfloat16*>(y1);
  if (x)
    repvgg_bwd_reduce_kernel<true><<<grid, kEwThreads, 0, st>>>(bg, ba, b3, b1, static_cast<const __nv_bfloat16*>(x), npix, C, s, sums);
  else
    repvgg_bwd_reduce_kernel<false><<<grid, kEwThreads, 0, st>>>(bg, ba, b3, b1, nullptr, npix, C, s, sums);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}

// count == nullptr: 1 / npix (this device's pixels); otherwise 1 / *count, the global count cvb_train_bn_merge left on the device
static int repvgg_bwd_apply(const void* g, const void* a, const void* y3, const void* y1, const void* x, int64_t npix, int32_t C, const RepvggStats& s,
                            const float* gamma3, const float* gamma1, const float* gamma_id, const float* sums, const double* count, void* dy3,
                            void* dy1, void* dx_id, cudaStream_t st) {
  const long long nvec = npix * (C / 8);
  const int grid = ew_grid(nvec);
  if (grid == 0) return CVB_ERR_NO_DEVICE;
  const auto* bg = static_cast<const __nv_bfloat16*>(g);
  const auto* ba = static_cast<const __nv_bfloat16*>(a);
  const auto* b3 = static_cast<const __nv_bfloat16*>(y3);
  const auto* b1 = static_cast<const __nv_bfloat16*>(y1);
  const auto* bx = static_cast<const __nv_bfloat16*>(x);
  auto* d3 = static_cast<__nv_bfloat16*>(dy3);
  auto* d1 = static_cast<__nv_bfloat16*>(dy1);
  auto* dx = static_cast<__nv_bfloat16*>(dx_id);
  const float inv_n = (float)(1.0 / (double)npix);
  if (x && count)
    repvgg_bwd_apply_kernel<true, true><<<grid, kEwThreads, 0, st>>>(bg, ba, b3, b1, bx, nvec, C, s, gamma3, gamma1, gamma_id, sums, 0.0f, count, d3, d1, dx);
  else if (x)
    repvgg_bwd_apply_kernel<true, false><<<grid, kEwThreads, 0, st>>>(bg, ba, b3, b1, bx, nvec, C, s, gamma3, gamma1, gamma_id, sums, inv_n, nullptr, d3, d1, dx);
  else if (count)
    repvgg_bwd_apply_kernel<false, true><<<grid, kEwThreads, 0, st>>>(bg, ba, b3, b1, nullptr, nvec, C, s, gamma3, gamma1, nullptr, sums, 0.0f, count, d3, d1,
                                                                      nullptr);
  else
    repvgg_bwd_apply_kernel<false, false><<<grid, kEwThreads, 0, st>>>(bg, ba, b3, b1, nullptr, nvec, C, s, gamma3, gamma1, nullptr, sums, inv_n, nullptr, d3,
                                                                       d1, nullptr);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}

extern "C" int cvb_train_repvgg_bwd(const void* g, const void* a, const void* y3, const void* y1, const void* x, int64_t npix, int32_t C,
                                    const float* stat3, const float* stat1, const float* stat_id, const float* gamma3, const float* gamma1,
                                    const float* gamma_id, float* sums, void* dy3, void* dy1, void* dx_id, void* stream) {
  CVB_REQUIRE(g && a && y3 && y1 && stat3 && stat1 && gamma3 && gamma1 && sums && dy3 && dy1, "train_repvgg_bwd: null pointer");
  const void* bf[] = {g, a, y3, y1, x, dy3, dy1, dx_id};
  const float* f32[] = {stat3, stat1, stat_id, gamma3, gamma1, gamma_id, sums};
  const int rc = check_repvgg("train_repvgg_bwd", npix, C, x, stat_id, bf, 8, f32, 7);
  if (rc != CVB_OK) return rc;
  CVB_REQUIRE((x == nullptr) == (gamma_id == nullptr) && (x == nullptr) == (dx_id == nullptr),
              "train_repvgg_bwd: x, stat_id, gamma_id and dx_id go together (all NULL: no identity branch)");
  cudaStream_t st = as_stream(stream);
  const RepvggStats s{stat3, stat1, stat_id};
  const int r = repvgg_bwd_reduce(g, a, y3, y1, x, npix, C, s, sums, st);
  return r != CVB_OK ? r : repvgg_bwd_apply(g, a, y3, y1, x, npix, C, s, gamma3, gamma1, gamma_id, sums, nullptr, dy3, dy1, dx_id, st);
}

// SyncBatchNorm halves of cvb_train_repvgg_bwd: one collective sums the [4][C] sums of all three branches over the ranks between them
extern "C" int cvb_train_repvgg_bwd_reduce(const void* g, const void* a, const void* y3, const void* y1, const void* x, int64_t npix, int32_t C,
                                           const float* stat3, const float* stat1, const float* stat_id, float* sums, void* stream) {
  CVB_REQUIRE(g && a && y3 && y1 && stat3 && stat1 && sums, "train_repvgg_bwd_reduce: null pointer");
  const void* bf[] = {g, a, y3, y1, x};
  const float* f32[] = {stat3, stat1, stat_id, sums};
  const int rc = check_repvgg("train_repvgg_bwd_reduce", npix, C, x, stat_id, bf, 5, f32, 4);
  if (rc != CVB_OK) return rc;
  return repvgg_bwd_reduce(g, a, y3, y1, x, npix, C, RepvggStats{stat3, stat1, stat_id}, sums, as_stream(stream));
}

extern "C" int cvb_train_repvgg_bwd_apply(const void* g, const void* a, const void* y3, const void* y1, const void* x, int64_t npix, int32_t C,
                                          const float* stat3, const float* stat1, const float* stat_id, const float* gamma3, const float* gamma1,
                                          const float* gamma_id, const float* sums, const double* count, void* dy3, void* dy1, void* dx_id,
                                          void* stream) {
  CVB_REQUIRE(g && a && y3 && y1 && stat3 && stat1 && gamma3 && gamma1 && sums && count && dy3 && dy1, "train_repvgg_bwd_apply: null pointer");
  const void* bf[] = {g, a, y3, y1, x, dy3, dy1, dx_id};
  const float* f32[] = {stat3, stat1, stat_id, gamma3, gamma1, gamma_id, sums};
  const int rc = check_repvgg("train_repvgg_bwd_apply", npix, C, x, stat_id, bf, 8, f32, 7);
  if (rc != CVB_OK) return rc;
  CVB_REQUIRE((x == nullptr) == (gamma_id == nullptr) && (x == nullptr) == (dx_id == nullptr),
              "train_repvgg_bwd_apply: x, stat_id, gamma_id and dx_id go together (all NULL: no identity branch)");
  CVB_REQUIRE(is_aligned(count, 8), "train_repvgg_bwd_apply: count must be 8-byte aligned");
  return repvgg_bwd_apply(g, a, y3, y1, x, npix, C, RepvggStats{stat3, stat1, stat_id}, gamma3, gamma1, gamma_id, sums, count, dy3, dy1, dx_id,
                          as_stream(stream));
}

extern "C" int cvb_train_convt_scatter(const void* u, int32_t B, int32_t h, int32_t w, int32_t C, const float* bias, void* out, void* stream) {
  CVB_REQUIRE(u && bias && out, "train_convt_scatter: null pointer");
  CVB_REQUIRE(B > 0 && h > 0 && w > 0 && C > 0 && C % 8 == 0, "train_convt_scatter: B, h, w must be > 0 and C a multiple of 8 (B=%d h=%d w=%d C=%d)", B,
              h, w, C);
  CVB_REQUIRE(is_aligned(u, 16) && is_aligned(out, 16) && is_aligned(bias, 4), "train_convt_scatter: u / out must be 16-byte, bias 4-byte aligned");
  const int grid = ew_grid((long long)B * 4 * h * w * (C / 8));
  if (grid == 0) return CVB_ERR_NO_DEVICE;
  convt_scatter_kernel<<<grid, kEwThreads, 0, as_stream(stream)>>>(static_cast<const __nv_bfloat16*>(u), B, h, w, C, bias, static_cast<__nv_bfloat16*>(out));
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return CVB_OK;
}

extern "C" int cvb_train_convt_gather(const void* g, int32_t B, int32_t h, int32_t w, int32_t C, float* scratch, void* du, float* dbias, void* stream) {
  CVB_REQUIRE(g && scratch && du && dbias, "train_convt_gather: null pointer");
  CVB_REQUIRE(B > 0 && h > 0 && w > 0 && C > 0 && C % 8 == 0 && C / 8 <= kEwThreads,
              "train_convt_gather: B, h, w must be > 0 and C a multiple of 8 up to 2048 (B=%d h=%d w=%d C=%d)", B, h, w, C);
  CVB_REQUIRE(is_aligned(g, 16) && is_aligned(du, 16) && is_aligned(scratch, 4) && is_aligned(dbias, 4),
              "train_convt_gather: g / du must be 16-byte, scratch / dbias 4-byte aligned");
  if (sm_count() == 0) return CVB_ERR_NO_DEVICE;
  cudaStream_t st = as_stream(stream);
  convt_gather_kernel<<<kConvtParts, kEwThreads, 0, st>>>(static_cast<const __nv_bfloat16*>(g), B, h, w, C, static_cast<__nv_bfloat16*>(du), scratch);
  convt_bias_finish_kernel<<<ceil_div(C, 128), 128, 0, st>>>(scratch, C, dbias);
  CVB_CHECK_CUDA(cudaGetLastError());
  count_launch(2);
  return CVB_OK;
}
