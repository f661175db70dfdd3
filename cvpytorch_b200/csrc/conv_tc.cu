// Fused conv2d + folded-BN bias + SiLU/ReLU (+ residual) (+ 2x-upsampled fp32 partial) for sm_90a (H100).
//
// Replaces the reference's per-layer chain  nn.Conv2d -> nn.BatchNorm2d -> nn.SiLU  (3 library kernels,
// src/models/bricks/conv_module.py:201-214; src/models/modules/yolo11_modules.py:27-39) plus the
// bottleneck shortcut add (src/models/modules/yolo_modules.py:95-104) and the neck's
// nearest-upsample + concat (src/models/modules/yolo11_modules.py:388-397) with ONE kernel.
//
// Formulation: implicit GEMM, NHWC.  D[128 pixels, BLOCK_N couts] += A[pixels, 64 cin] * W[couts, 64 cin]^T per
// (filter tap, cin chunk).  A tile = a TMA box {BLOCK_K channels, TW, TH, NB} of the input tensor shifted by
// the tap offset; TMA's out-of-bounds zero fill IS the convolution padding.  Stride-2 convolutions read
// through four "parity" tensor maps (even/odd rows x even/odd columns), so the kernel never sees the stride.
//
// Precision: activations/weights are fp16 (hi, lo) pairs; three wgmma per K step
// (hi*hi + hi*lo + lo*hi), fp32 accumulation in registers -> fp32-equivalent results (rel. err ~1e-6) on the
// fp16 tensor pipe.  The reference computes fp32 (trainer.py:209 val path is un-autocast).
//
// Structure (persistent, warp specialised, 288 threads, 1 or 2 CTAs/SM):
//   warp 8      TMA producer   (one lane)   smem ring: full[]/empty[] mbarriers
//   warps 0..7  two warpgroups: wgmma main loop over the ring (warpgroup w owns accumulator rows 64w..64w+63), then the epilogue:
//               registers -> fp32 shared-memory tile (one output group at a time) -> +partial +bias -> act -> +residual -> hi/lo split
//               -> swizzled smem -> TMA store
#include <cuda_fp16.h>
#include <math_constants.h>

#include <cstdlib>
#include <memory>
#include <new>
#include <type_traits>

#include "internal.h"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace cvb {

#ifndef CVB_DIAG
#define CVB_DIAG 0  // 1: the per-role cycle counters (cvb_conv_plan_set_profile) and the CVB_DBG switches are compiled in (tools build: libcvb200_diag.so)
#endif
constexpr bool kDiag = CVB_DIAG != 0;
constexpr int kTileM = 128;
constexpr int kMaxTaps = 9;
constexpr int kEpiThreads = 256;          // two MMA / epilogue warpgroups
constexpr int kMmaWarps = kEpiThreads / 32;
constexpr int kProducerWarp = kMmaWarps;  // the TMA producer warp follows the warpgroups
constexpr int kThreads = kEpiThreads + 32;
constexpr int kYoloBiasBytes = 4 * 128 * 4;  // fused decode: bias of all (<= 4) anchors, loaded once per CTA
constexpr int kYoloStageBytes = 45056;  // fused decode: [128][85] fp32 staging tile + 3 x 128 partial row maxima, rounded to 1 KB
constexpr int kSmemBudget = 232448;  // 227 KB opt-in limit per CTA on sm_90
constexpr int kSmemBudget2 = 115712;  // per CTA when two share an SM: (228 KB - 2 x 1 KB reserved) / 2
constexpr int kMaxBars = 64;                  // mbarrier slots of a CTA
constexpr int kBarBytes = kMaxBars * 8 + 16;  // mbarrier area

// Per-tile shared-memory geometry of a kernel instantiation: the kernel's compile-time constants, and what the planner sizes plans with.
// pp: ping-pong schedule -- a tile is 64 pixels and belongs to one warpgroup, so every per-tile buffer exists once per warpgroup.
struct ConvGeom {
  int tile_m;           // output pixels of one tile
  int swz;              // swizzle span == bytes of one K chunk row
  int a_bytes, b_bytes; // one plane of the activation / weight tile of one K chunk
  int out_group_ch, out_row_bytes, out_plane_bytes;
  int out_tile_bytes;   // staging tile of one output group of one tile
  int out_buf_bytes;  // one staging buffer (ping-pong: one tile per warpgroup)
  int acc_pitch, acc_bytes;
  int bias_bytes;
};
__host__ __device__ constexpr ConvGeom conv_geom(int block_n, int block_k, bool f32, bool yolo, bool pp) {
  const int tile_m = pp ? kTileM / 2 : kTileM;
  const int gch = f32 ? 32 : (block_n >= 64 ? 64 : 32);
  const int row = f32 ? 128 : gch * 2;
  const int tile = tile_m * row * (f32 ? 1 : 2);
  // fp32 accumulator tile the epilogue reads (one output group, or the 96 decoded columns of a fused-decode tile); rows padded by
  // 16 bytes so that the row-per-thread reads of eight consecutive rows hit distinct banks.  Ping-pong: rows 64*wg.. are warpgroup wg's tile.
  const int acc_pitch = (yolo ? 96 : gch) + 4;
  return ConvGeom{tile_m, block_k * 2, tile_m * block_k * 2, block_n * block_k * 2, gch, row, tile_m * row, tile, tile * (pp ? 2 : 1),
                  acc_pitch, kTileM * acc_pitch * 4, (pp ? 2 : 1) * block_n * 4};
}

// Byte offsets of the regions of a CTA's dynamic shared memory, in address order; the ring starts at offset 0.  smem_layout builds it on
// the host.  The plan carries it in ConvKArgs::sm: the kernel reads the ring slot, and the diagnostics build checks its region pointers
// against the offsets.
struct SmemLayout {
  int slot;     // bytes of one ring slot
  int weights;  // resident weight slab, or the halo loader's weight ring
  int out;      // output staging tiles (fused decode: staging tile, NMS histogram and bias)
  int resid;    // residual staging tile
  int acc;      // fp32 accumulator tile
  int bias;     // bias of the current n-tile
  int bars;     // mbarriers
  int total;
};

struct alignas(64) ConvKArgs {
  CUtensorMap tmA[4];  // input, one per (row parity, col parity) for stride 2; only [0] for stride 1
  CUtensorMap tmB;     // weights [2][cout_pad][K]
  CUtensorMap tmO;     // output (5D; plane dim = 1 for fp32)
  CUtensorMap tmR;     // residual (same box as the output tile), loaded by TMA into a staging tile
  int tiles_w, tiles_h, tiles_b, tiles_n;
  uint32_t mg_n, mg_w, mg_h;   // fast_div_magic of tiles_{n,w,h}: tile index -> coordinates by multiply-high
  int TW, TH, NB;
  int Ho, Wo, Bn;
  int cout;
  int taps, chunks, cin;
  int stages;
  int act;
  int rows_valid;
  uint32_t a_box_bytes;
  uint32_t a_lo_off;   // smem offset of the lo plane of A inside a stage (== a_box_bytes when hi+lo arrive in ONE TMA box)
  int a_fused;         // 1: one 5D box {K, TW, TH, NB, 2 planes} per stage instead of two
  int b_resident;      // 1: the whole weight slab of this CTA's n-tile stays in smem; the ring streams A only
  int resid_tma;       // 1: the residual tile arrives by TMA (issued one group ahead by the epilogue), 0: per-thread loads
  int resid_first;     // 1: out = act(conv + bias + residual) (ResNet bottleneck); 0: out = act(conv + bias) + residual (Darknet)
  float resid_scale;   // weight of the residual operand (1 for the Darknet / ResNet shortcuts, alpha of the YOLOv6 BottleRep)
  float rz_gain;       // 1 + (MMAs per hi*hi chain) * c: undoes the mean shrink of round-toward-zero accumulation (see DESIGN.md 2)
  int out_bufs;        // 1 or 2 output staging tiles (2: the TMA store of group g overlaps the conversion of g+1)
  int8_t tap_map[kMaxTaps];
  int8_t tap_dh[kMaxTaps];
  int8_t tap_dw[kMaxTaps];
  const float* bias;
  int bias_len;
  const __half* resid;
  long long resid_plane;  // elements
  int resid_pitch;        // elements per pixel
  const float* up;
  int up_pitch, up_H, up_W;
  // ---- "halo" (copy / tap) mode: the activation tile is loaded ONCE per K chunk as one or a few boxes that include the filter
  // halo ("copies"), and every filter tap is a row-shifted shared-memory descriptor view of a copy -- instead of one TMA box per tap.
  // Cuts the L2 -> shared-memory fill traffic of a 3x3 layer up to 6x (the chip-wide L2 fill rate bounds those layers, DESIGN.md 4.1).
  int halo;              // 0: classic, 1: one copy per horizontal tap offset (aligned views), 2: one copy per input map (full halo)
  int n_copies;
  int sb_stages;         // depth of the separate weight-tile ring (0: weights resident)
  int kskip;             // K steps (of 16) skipped at the end of every chunk (zero weight columns of the row-window stems)
  uint32_t cp_bytes[6];  // bytes of ONE plane of copy c
  uint32_t cp_lo_off[6]; // offset of the lo plane inside the slot
  uint32_t cp_sbo[6];    // byte stride between the 8-row groups of a tap view of copy c (= one row of the copy's halo image)
  uint16_t tap_off[kMaxTaps];  // first row of the tap's view inside its copy
  int8_t cp_map[6], cp_dw[6], cp_dh[6], cp_ntaps[6];
  int8_t tap_w[kMaxTaps];      // index of the tap in the packed weights (ky * kw + kx)
  // the taps of copy c form an ny x nx grid: view offset = y * cp_row16 + x * (row bytes >> 4) (16-byte units), weight tap = w0 + y*wy + x*wx
  uint32_t cp_row16[6];
  int8_t cp_ny[6], cp_nx[6], cp_w0[6], cp_wy[6], cp_wx[6];
  // ---- fused YOLOv5 decode epilogue (YOLO kernels): n-tile = anchor (85 of 128 columns used), z rows / NMS histogram / rowmax written directly
  int tile_contig;             // 1: every CTA owns a contiguous run of tiles (image-major), so its shared-memory histogram belongs to <= 2 images
  float* yz;                   // z [B, y_zrows, y_no] fp32
  long long y_zrows, y_zoff;
  int y_no, y_multi;
  int y_nx;                    // level width (the conv itself runs on the flattened level: Wo = ny * nx, Ho = 1)
  uint32_t y_nx_magic;         // ceil(2^32 / nx): pixel -> row by multiply-high
  float y_stride, y_conf;
  float y_anchor[8];           // anchor sizes in pixels: [a * 2 + 0] = w, [a * 2 + 1] = h
  unsigned int* y_hist;        // NMS workspace histogram [B][kNmsBins] (or NULL)
  float* y_rowmax;             // NMS workspace per-row best score [B][y_zrows] (or NULL)
  uint32_t wait_hint;          // suspend-time hint (ns) of the producer's free-slot waits (CVB_WAIT_HINT, 0 = spin)
  int dbg;                     // diagnostics (CVB_DBG, results are WRONG): bit 0 = no TMA stores, bit 1 = activations loaded only for the first ring pass, bit 2 = epilogue skips the math / staging, bit 5 = fused decode without histogram atomics, bit 6 = without the z copy-out, bits 10 / 11 = classic loader streams weight tiles on every other ring fill / the first ring pass only
  long long* prof;             // diagnostics (cvb_conv_plan_set_profile): per-CTA cycle counters of the three pipeline roles, or NULL
  SmemLayout sm;
};

// first output column, row, image and channel of a tile; tile = ((bt * tiles_h + ht) * tiles_w + wt) * tiles_n + nt
struct TileOrigin {
  int w0, h0, b0, n0;
};
template <int BLOCK_N>
__device__ __forceinline__ TileOrigin tile_origin(const ConvKArgs& a, int tile) {
  const int mt = fast_div(tile, a.tiles_n, a.mg_n), nt = tile - mt * a.tiles_n;
  const int t2 = fast_div(mt, a.tiles_w, a.mg_w), wt = mt - t2 * a.tiles_w;
  const int bt = fast_div(t2, a.tiles_h, a.mg_h), ht = t2 - bt * a.tiles_h;
  return TileOrigin{wt * a.TW, ht * a.TH, bt * a.NB, nt * BLOCK_N};
}

__device__ __forceinline__ float apply_act(float x, int act) {
  if (act == CVB_ACT_SILU) return __fdividef(x, 1.0f + __expf(-x));
  if (act == CVB_ACT_RELU) return fmaxf(x, 0.0f);
  return x;
}

// x * sigmoid(x) with two MUFU ops (ex2, rcp); |rel err| ~ 2^-22.  x -> -inf gives -0, x -> +inf gives x.
__device__ __forceinline__ float silu_fast(float x) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * -1.4426950408889634f));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
  return x * r;
}

// diagnostics: cycles spent in a waiting primitive, accumulated per role (only when a profile buffer is attached)
#define CVB_PROF_WAIT(slot, stmt)              \
  do {                                         \
    if (prof_on) {                             \
      const long long _t0 = clock64();         \
      stmt;                                    \
      prof_acc[slot] += clock64() - _t0;       \
    } else {                                   \
      stmt;                                    \
    }                                          \
  } while (0)

__device__ __forceinline__ uint64_t desc64(uint32_t lo, uint32_t hi) { return ((uint64_t)hi << 32) | lo; }

// The MMAs of one (filter tap, K chunk) for the 64 accumulator rows of this warpgroup: KSTEPS K steps of 16 over the hi / lo
// activation views and the hi / lo weight tiles.  SPLIT: hi*hi -> dm, the (2^-11 smaller) cross terms hi*lo + lo*hi -> dc; else all
// three products -> dm (the 256-wide tiles, whose two accumulators would not fit the register file).
// Descriptor low words in 16-byte units (a16: hi activation view, a16 + lo16: lo view, b16: hi weight tile, + bl16: lo tile); the
// high words are loop invariants.
// PRED: only the first `ksteps` K steps are issued (the halo loader's row-window stems skip their zero weight columns).  The run-time
// predicate between the wgmmas of a tap makes ptxas fence the accumulator registers (warpgroup.arrive, C7519) before every K step, so the
// ping-pong kernels, which have no halo loader, issue the KSTEPS steps as one straight wgmma sequence.  The cooperative kernels keep it:
// without it ptxas serializes their wgmmas (C7515), which costs more than the fences.
template <int BLOCK_N, int KSTEPS, bool SPLIT, bool PRED>
__device__ __forceinline__ void issue_tap(float (&dm)[BLOCK_N / 2], float (&dc)[SPLIT ? BLOCK_N / 2 : 1], uint32_t a16, uint32_t lo16,
                                          uint32_t a_hi, uint32_t b16, uint32_t bl16, uint32_t b_hi, int ksteps) {
#pragma unroll
  for (int k = 0; k < KSTEPS; ++k) {
    if (!PRED || k < ksteps) {
      const uint64_t ah = desc64(a16 + 2 * k, a_hi), al = desc64(a16 + lo16 + 2 * k, a_hi);
      const uint64_t bh = desc64(b16 + 2 * k, b_hi), bl = desc64(b16 + bl16 + 2 * k, b_hi);
      wgmma_m64k16<BLOCK_N, 0, 0>(dm, ah, bh);
      if constexpr (SPLIT) {
        wgmma_m64k16<BLOCK_N, 0, 0>(dc, ah, bl);
        wgmma_m64k16<BLOCK_N, 0, 0>(dc, al, bh);
      } else {
        wgmma_m64k16<BLOCK_N, 0, 0>(dm, ah, bl);
        wgmma_m64k16<BLOCK_N, 0, 0>(dm, al, bh);
      }
    }
  }
}

// EPI selects a compile-time specialisation of the epilogue (the hot layers run a compact, branch-free instruction stream; the generic
// stream with its run-time mode checks costs more issue slots per tile, and the HBM-bound layers are issue bound in the epilogue):
//   0 generic   1 act = SiLU, no residual, no up-partial   2 act = SiLU, residual tile by TMA added after the activation (Darknet bottleneck)
//   3 act = ReLU, no residual, no up-partial   4 act = ReLU, residual tile by TMA added BEFORE the activation (ResNet bottleneck)
// PP selects the ping-pong schedule (one-CTA-per-SM plans, not for the fused decode or the halo loader): a tile is 64 pixels, the
// CTA's tiles alternate between the two warpgroups, and a warpgroup runs its epilogue while the other one's MMAs run (DESIGN.md 4.1).
// CTAS: the CTAs per SM the register budget is sized for.  Only the cooperative narrow kernels may share an SM, and they exist with both
// bounds: the two-CTA plans need the 96-register cap, the one-CTA plans would spill under it for nothing.  A ping-pong plan always runs
// one CTA per SM and gets the full register budget.
template <int BLOCK_N, int BLOCK_K, bool OUT_F32, bool YOLO, int EPI = 0, bool PP = false, int CTAS = 1>
__global__ void __launch_bounds__(kThreads, CTAS) conv_tc_kernel(const __grid_constant__ ConvKArgs a) {
  constexpr ConvGeom G = conv_geom(BLOCK_N, BLOCK_K, OUT_F32, YOLO, PP);
  constexpr int SWZ = G.swz;
  constexpr int A_BYTES = G.a_bytes;
  constexpr int B_BYTES = G.b_bytes;
  constexpr int OUT_GROUP_CH = G.out_group_ch;
  constexpr int OUT_ROW_BYTES = G.out_row_bytes;
  constexpr int OUT_PLANE_BYTES = G.out_plane_bytes;
  constexpr int OUT_TILE_BYTES = G.out_tile_bytes;
  constexpr int ACC_PITCH = G.acc_pitch;
  // ring slots, weight tiles and staging tiles are multiples of the 1024-byte swizzle atom, so every TMA-swizzled region the host lays
  // out starts on a 1024-byte boundary
  static_assert(A_BYTES % 1024 == 0 && B_BYTES % 1024 == 0 && OUT_TILE_BYTES % 1024 == 0, "swizzled tiles must be 1024-byte multiples");
  constexpr int EPI_THREADS = PP ? kEpiThreads / 2 : kEpiThreads;  // threads that share one tile's epilogue
  constexpr bool SPLIT = BLOCK_N <= 128;
  static_assert(EPI == 0 || (!OUT_F32 && !YOLO), "epilogue specialisations exist for the split16 output only");
  static_assert(!(PP && YOLO), "the fused decode runs the cooperative schedule");
  static_assert(CTAS == 1 || (CTAS == 2 && BLOCK_N <= 64 && !PP && !YOLO), "only the cooperative narrow kernels may share an SM");
  // run-time mode flags, folded to constants in the specialised kernels
  const bool resid_tma = (EPI == 2 || EPI == 4) ? true : ((EPI == 1 || EPI == 3) ? false : a.resid_tma != 0);
  const int act_mode = (EPI == 1 || EPI == 2) ? CVB_ACT_SILU : ((EPI == 3 || EPI == 4) ? CVB_ACT_RELU : a.act);

  // the kernel has no static shared memory, so the dynamic window starts at offset 0 of the CTA's (1024-byte aligned)
  // allocation; checked once instead of spending 1 KB of slack (which is what lets some two-CTA plans fit in 113 KB)
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw;
  if (threadIdx.x == 0 && (smem_u32(smem) & 1023u) != 0u) {
    printf("conv_tc_kernel: dynamic shared memory is not 1024-byte aligned\n");
    __trap();
  }
  const int dbg = kDiag ? a.dbg : 0;  // diagnostics switches: compiled out of the product library
  const int STAGES = a.stages;
  const bool halo = PP ? false : a.halo != 0;
  // Region pointers in smem_layout's order, chained from the plan's ring / weight / staging parameters and the compile-time geometry.
  // Taking them from a.sm, or from smem_layout made a __host__ __device__ function, costs registers at the 168-register cap: ptxas adds
  // spills to 23 to 53 of the instantiations.  The diagnostics build checks the chain against the plan's offsets.
  const int stage_bytes = halo ? (int)a.sm.slot : (a.b_resident ? 2 * A_BYTES : 2 * A_BYTES + 2 * B_BYTES);
  uint8_t* stage_base = smem;
  uint8_t* b_res = smem + STAGES * stage_bytes;
  uint8_t* out_stage0 = b_res + (a.b_resident ? a.taps * a.chunks * 2 * B_BYTES : (halo ? a.sb_stages * 2 * B_BYTES : 0));
  uint8_t* res_stage = out_stage0 + (YOLO ? kYoloStageBytes + kNmsBins * 4 + kYoloBiasBytes : a.out_bufs * G.out_buf_bytes);
  float* acc_s = reinterpret_cast<float*>(res_stage + (resid_tma ? G.out_buf_bytes : 0));
  float* bias_s = acc_s + G.acc_bytes / 4;
  uint64_t* bars = reinterpret_cast<uint64_t*>(bias_s + (PP ? 2 : 1) * BLOCK_N);
  if (kDiag && threadIdx.x == 0 &&
      (b_res != smem + a.sm.weights || out_stage0 != smem + a.sm.out || res_stage != smem + a.sm.resid ||
       reinterpret_cast<uint8_t*>(acc_s) != smem + a.sm.acc || reinterpret_cast<uint8_t*>(bias_s) != smem + a.sm.bias ||
       reinterpret_cast<uint8_t*>(bars) != smem + a.sm.bars || stage_bytes != a.sm.slot)) {
    // (no printf here: its call makes ptxas serialize every wgmma of the diagnostics build, which then times a different main loop)
    __trap();  // shared-memory regions differ from the plan's layout
  }
  const int SB = halo ? a.sb_stages : 0;
  uint64_t* full = bars;
  uint64_t* empty = bars + STAGES;
  uint64_t* fullB = bars + 2 * STAGES;  // halo mode: separate ring of weight tiles
  uint64_t* emptyB = fullB + SB;
  uint64_t* bfull = emptyB + SB;  // resident weights have landed
  uint64_t* rfull = bfull + 1;    // residual tile has landed (ping-pong: one per warpgroup)

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == kProducerWarp && lane == 0) {
    tma_prefetch_desc(&a.tmA[0]);
    tma_prefetch_desc(&a.tmB);
    if constexpr (!YOLO) tma_prefetch_desc(&a.tmO);
    if (resid_tma) tma_prefetch_desc(&a.tmR);
  }
  if (threadIdx.x == 0) {
    // a ring slot is free once every MMA warp that reads it has seen its wgmma group complete (ping-pong: the 4 warps of one warpgroup)
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], PP ? kMmaWarps / 2 : kMmaWarps);
    }
    for (int s = 0; s < SB; ++s) {
      mbar_init(&fullB[s], 1);
      mbar_init(&emptyB[s], kMmaWarps);
    }
    mbar_init(bfull, 1);
    mbar_init(rfull, 1);
    if (PP) mbar_init(rfull + 1, 1);
    fence_barrier_init();
  }
  __syncthreads();
  // Programmatic dependent launch: everything above (barrier init, descriptor prefetch) and the resident weight load below touch only
  // this kernel's own state or static data, so it may overlap the previous kernel's tail.
  grid_dep_launch_dependents();

  const int m_tiles = a.tiles_w * a.tiles_h * a.tiles_b;
  const int total_tiles = m_tiles * a.tiles_n;
  const int k_iters = a.taps * a.chunks;
  // tiles of this CTA: strided over the grid (default), or one contiguous run (fused-decode kernels: image-major order keeps the CTA's
  // shared-memory NMS histogram on one or two images)
  int t_begin = (int)blockIdx.x, t_end = total_tiles, t_step = (int)gridDim.x;
  if (a.tile_contig) {
    const int per = (total_tiles + (int)gridDim.x - 1) / (int)gridDim.x;
    t_begin = (int)blockIdx.x * per;
    t_end = min(total_tiles, t_begin + per);
    t_step = 1;
  }
  // Tile order: tile = mt * tiles_n + nt.  Every CTA strides by gridDim.x; in resident mode gridDim.x is a multiple of
  // tiles_n, so nt = tile % tiles_n is the same for all tiles of a CTA and its weight slab is loaded exactly once.

  if (warp == kProducerWarp) {
    // ------------------------------------------------------------------ TMA producer
    if (elect_one() && !(dbg & 16)) {
      const bool prof_on = kDiag && a.prof != nullptr;
      long long prof_acc[4] = {0, 0, 0, 0};
      const long long prof_t0 = prof_on ? clock64() : 0;
      int stage = 0;
      uint32_t phase = 0;
      const uint32_t tx_bytes = 2 * a.a_box_bytes + (a.b_resident ? 0 : 2 * B_BYTES);
      if (a.b_resident && t_begin < t_end) {
        const int n0r = ((int)blockIdx.x % a.tiles_n) * BLOCK_N;
        mbar_expect_tx(bfull, (uint32_t)(k_iters * 2 * B_BYTES));
        for (int it = 0; it < k_iters; ++it) {
          const int tap = it / a.chunks, ck = it - tap * a.chunks;
          tma_load_3d(&a.tmB, bfull, b_res + it * 2 * B_BYTES, tap * a.cin + ck * BLOCK_K, n0r, 0);
        }
      }
      grid_dep_wait();  // activations are written by the previous kernel(s)
      if (halo) {
        // copy / tap mode: per (tile, K chunk) one box per copy (all filter rows -- and in mode 2 all filter columns -- of that
        // chunk), then the weight tiles of the copy's taps in the order the MMA warp consumes them
        int sb = 0;
        uint32_t phase_b = 0;
        for (int tile = t_begin; tile < t_end; tile += t_step) {
          const TileOrigin to = tile_origin<BLOCK_N>(a, tile);
          const int w0 = to.w0, h0 = to.h0, b0 = to.b0, n0 = to.n0;
          for (int ck = 0; ck < a.chunks; ++ck) {
            int t = 0;
            for (int c = 0; c < a.n_copies; ++c) {
              CVB_PROF_WAIT(0, mbar_wait(&empty[stage], phase ^ 1, 100 + stage, a.wait_hint));
              if ((dbg & 2) && (tile != t_begin)) {
                mbar_arrive(&full[stage]);  // diagnostics: no data movement after the first tile
              } else {
              mbar_expect_tx(&full[stage], 2 * a.cp_bytes[c]);
              uint8_t* sb_a = stage_base + stage * stage_bytes;
              const CUtensorMap* mapA = &a.tmA[a.cp_map[c]];
              tma_load_5d(mapA, &full[stage], sb_a, ck * BLOCK_K, w0 + a.cp_dw[c], h0 + a.cp_dh[c], b0, 0);
              if (!a.a_fused) tma_load_5d(mapA, &full[stage], sb_a + a.cp_lo_off[c], ck * BLOCK_K, w0 + a.cp_dw[c], h0 + a.cp_dh[c], b0, 1);
              }
              if (++stage == STAGES) {
                stage = 0;
                phase ^= 1;
              }
              if (!a.b_resident) {
                for (int j = 0; j < a.cp_ntaps[c]; ++j, ++t) {
                  CVB_PROF_WAIT(1, mbar_wait(&emptyB[sb], phase_b ^ 1, 150 + sb, a.wait_hint));
                  mbar_expect_tx(&fullB[sb], 2 * B_BYTES);
                  tma_load_3d(&a.tmB, &fullB[sb], b_res + sb * 2 * B_BYTES, a.tap_w[t] * a.cin + ck * BLOCK_K, n0, 0);
                  if (++sb == SB) {
                    sb = 0;
                    phase_b ^= 1;
                  }
                }
              }
            }
          }
        }
      } else
      for (int tile = t_begin, fill = 0; tile < t_end; tile += t_step) {
        const TileOrigin to = tile_origin<BLOCK_N>(a, tile);
        const int w0 = to.w0, h0 = to.h0, b0 = to.b0, n0 = to.n0;
        for (int tap = 0; tap < a.taps; ++tap) {
          const CUtensorMap* mapA = &a.tmA[a.tap_map[tap]];
          const int cw = w0 + a.tap_dw[tap];
          const int ch = h0 + a.tap_dh[tap];
          for (int ck = 0; ck < a.chunks; ++ck, ++fill) {
            CVB_PROF_WAIT(0, mbar_wait(&empty[stage], phase ^ 1, 100 + stage, a.wait_hint));
            // diagnostics: streamed weight tiles on every other ring fill only (bit 10: half the weight traffic from L2), or on the
            // first ring pass only (bit 11); the other fills reuse whatever the slot holds
            const bool cut_b = kDiag && !a.b_resident && (((dbg & 1024) && (fill & 1)) || ((dbg & 2048) && fill >= STAGES));
            mbar_expect_tx(&full[stage], cut_b ? 2 * a.a_box_bytes : tx_bytes);
            uint8_t* sb = stage_base + stage * stage_bytes;
            tma_load_5d(mapA, &full[stage], sb, ck * BLOCK_K, cw, ch, b0, 0);  // fused: both planes in one box
            if (!a.a_fused) tma_load_5d(mapA, &full[stage], sb + A_BYTES, ck * BLOCK_K, cw, ch, b0, 1);
            if (!a.b_resident && !cut_b) {
              const int kc = tap * a.cin + ck * BLOCK_K;
              tma_load_3d(&a.tmB, &full[stage], sb + 2 * A_BYTES, kc, n0, 0);  // box {K, N, 2 planes}: hi then lo
            }
            if (++stage == STAGES) {
              stage = 0;
              phase ^= 1;
            }
          }
        }
      }
      if (prof_on) {  // producer: total cycles, waiting for a free A slot, waiting for a free weight slot (ping-pong: in both counter rows)
        const long long t = clock64() - prof_t0;
        for (int r = 0; r < (PP ? 2 : 1); ++r) {
          long long* pr = a.prof + ((size_t)r * gridDim.x + blockIdx.x) * 16;
          pr[0] = t;
          pr[1] = prof_acc[0];
          pr[2] = prof_acc[1];
        }
      }
    }
  } else {
    // ------------------------------------------------------------------ MMA + epilogue (warps 0..7: two warpgroups)
    // Warpgroup wg issues the wgmmas of accumulator rows 64*wg .. +63 of every tile (register accumulators), then all eight warps
    // run the epilogue from a shared-memory copy of the accumulators; the producer warp keeps the ring full meanwhile.
    // Ping-pong: warpgroup wg owns every other tile of the CTA (64 pixels, all BLOCK_N columns) and runs its MMAs and its epilogue
    // alone, with its own accumulator rows 64*wg.., staging tiles, residual tile, bias and epilogue barrier.
    const int wg = warp >> 2;
    // fused decode: the rows of warpgroup wg are decode group wg (its staging half, barrier and bulk store); plain epilogue: two warps
    // per row quarter (ping-pong: per row half), each converting half of the columns of every staged group
    const int q = warp & 3;
    const int half = YOLO ? ((warp >> 1) & 1) : (PP ? (q >> 1) : (warp >> 2));
    const int row = YOLO ? 64 * wg + 32 * (warp & 1) + lane : (PP ? (q & 1) * 32 + lane : q * 32 + lane);  // pixel index inside the tile box
    const int tid_e = PP ? (int)threadIdx.x & (EPI_THREADS - 1) : (int)threadIdx.x;
    const int ebar = PP ? 2 + wg : 1;                                         // epilogue barrier of the tile's EPI_THREADS threads
    float* const acc_t = acc_s + (PP ? 64 * wg * ACC_PITCH : 0);               // accumulator rows of the tile
    float* const bias_t = bias_s + (PP ? wg * BLOCK_N : 0);
    uint64_t* const rfull_t = rfull + (PP ? wg : 0);
    uint8_t* const res_t = res_stage + (PP ? wg * OUT_TILE_BYTES : 0);
    const int tw = row % a.TW;
    const int r2 = row / a.TW;
    const int th = r2 % a.TH;
    const int nb = r2 / a.TH;
    constexpr int CW = OUT_GROUP_CH / 2;  // columns per warp per group (32, or 16 for 32-wide groups)
    constexpr int SUB = (BLOCK_N <= 64 && CW > 16) ? 16 : CW;  // columns held in registers at a time
    const bool prof_on = kDiag && a.prof != nullptr;
    long long prof_acc[6] = {0, 0, 0, 0, 0, 0};
    const long long prof_t0 = prof_on ? clock64() : 0;

    // ---- main loop state (persists across tiles: the ring positions of the producer)
    int stage = 0;
    uint32_t phase = 0;
    int hb = 0;  // halo mode: weight ring position
    uint32_t hphase_b = 0;
    // shared-memory descriptor words (see make_kmajor_desc): low word = start address >> 4 | LBO 1 << 16; high word = SBO >> 4 |
    // swizzle layout << 29.  Everything below is kept in 16-byte units so that one 32-bit add moves a view.
    constexpr int KSTEPS = BLOCK_K / 16;
    constexpr uint32_t kLayout = SWZ == 128 ? 2u : (SWZ == 64 ? 4u : 6u);
    constexpr uint32_t kHiStd = ((8u * SWZ) >> 4) | (kLayout << 29);
    constexpr uint32_t kB16 = (uint32_t)B_BYTES >> 4;
    const uint32_t ring16 = ((smem_u32(stage_base) & 0x3FFFFu) >> 4) | 0x10000u;
    const uint32_t bres16 = ((smem_u32(b_res) & 0x3FFFFu) >> 4) | 0x10000u;
    const uint32_t stage16 = (uint32_t)stage_bytes >> 4;
    const bool resident = a.b_resident != 0;
    const int ksteps = KSTEPS - a.kskip;
    const int chunks = a.chunks;
    uint32_t a_ring16 = ring16;  // descriptor low word of the current A slot / stage
    float dm[BLOCK_N / 2];
    float dc[SPLIT ? BLOCK_N / 2 : 1];
    // Ring slots whose wgmmas are in flight: a unit's slots are released once the NEXT unit has been issued and the unit itself has
    // completed (wgmma.wait_group 1), so the tensor pipe always has the next unit queued.
    int pend_a = -1, pend_b = -1;
    auto unit_issued = [&](int a_slot, int b_slot) {
      wgmma_commit();
      wgmma_wait<1>();
      wgmma_fence_regs(dm);
      if constexpr (SPLIT) wgmma_fence_regs(dc);
      if (lane == 0) {
        if (pend_a >= 0) mbar_arrive(&empty[pend_a]);
        if (pend_b >= 0) mbar_arrive(&emptyB[pend_b]);
      }
      pend_a = a_slot;
      pend_b = b_slot;
    };
    // One tile: dm = gain * (hi*hi chain) + cross terms.  The tensor core's fp32 adder rounds toward zero, so a long accumulation chain
    // shrinks |sum| slightly per MMA; rz_gain undoes the mean shrink and the (2^-11 smaller) cross terms have their own accumulator.
    // Ping-pong: `pass_turn` hands the tensor pipe to the other warpgroup (named barrier 4 + other) once every MMA of the tile has been
    // issued, before this warpgroup waits for them to complete.
    auto mainloop = [&](bool pass_turn) {
#pragma unroll
      for (int i = 0; i < BLOCK_N / 2; ++i) dm[i] = 0.0f;
      if constexpr (SPLIT) {
#pragma unroll
        for (int i = 0; i < BLOCK_N / 2; ++i) dc[i] = 0.0f;
      }
      if (halo) {
        // copy / tap mode: every tap is a row-shifted descriptor view of the copy in the current A slot; weight tiles come from the
        // resident slab or from their own ring.  The taps of a copy form an ny x nx grid (filter rows x filter columns) whose view
        // offsets and weight indices are affine in (y, x): two running descriptor words, no per-tap table.
        const uint32_t wstep16 = (uint32_t)chunks * 2u * kB16;  // resident slab: distance between consecutive weight taps
        for (int ck = 0; ck < chunks; ++ck) {
          for (int c = 0; c < a.n_copies; ++c) {
            const int ny = a.cp_ny[c], nx = a.cp_nx[c];
            const uint32_t row16 = a.cp_row16[c], lo16 = a.cp_lo_off[c] >> 4;
            const uint32_t a_hi = (a.cp_sbo[c] >> 4) | (kLayout << 29);
            const uint32_t wy16 = (uint32_t)a.cp_wy[c] * wstep16, wx16 = (uint32_t)a.cp_wx[c] * wstep16;
            uint32_t brow16 = bres16 + (uint32_t)a.cp_w0[c] * wstep16 + (uint32_t)ck * 2u * kB16;
            mbar_wait(&full[stage], phase, 300 + stage);
            // rows 64*wg.. of a tap view = output rows 8*wg.. of the 8 x 16 tile: 8 halo rows (of cp_sbo bytes) further
            uint32_t arow16 = a_ring16 + (uint32_t)wg * (a.cp_sbo[c] >> 1);
            for (int y = 0; y < ny; ++y, arow16 += row16, brow16 += wy16) {
              uint32_t a16 = arow16, b16 = brow16;
              for (int x = 0; x < nx; ++x, a16 += (SWZ >> 4), b16 += wx16) {
                uint32_t bb = b16;
                if (!resident) {
                  mbar_wait(&fullB[hb], hphase_b, 350 + hb);
                  bb = bres16 + (uint32_t)hb * 2u * kB16;
                }
                wgmma_fence();
                issue_tap<BLOCK_N, KSTEPS, SPLIT, !PP>(dm, dc, a16, lo16, a_hi, bb, kB16, kHiStd, ksteps);
                // the A slot is released with the last tap of the copy, the weight slot with its tap
                unit_issued((y == ny - 1 && x == nx - 1) ? stage : -1, resident ? -1 : hb);
                if (!resident && ++hb == SB) {
                  hb = 0;
                  hphase_b ^= 1;
                }
              }
            }
            a_ring16 += stage16;
            if (++stage == STAGES) {
              stage = 0;
              phase ^= 1;
              a_ring16 = ring16;
            }
          }
        }
      } else {
        const uint32_t lo16 = a.a_lo_off >> 4;
        const uint32_t wg16 = PP ? 0u : (uint32_t)wg * (4u * SWZ);  // rows 64*wg..: eight 8-row groups of 8 * SWZ bytes
        uint32_t bres_it16 = bres16;
        for (int i = 0; i < k_iters; ++i, bres_it16 += 2u * kB16) {
          CVB_PROF_WAIT(5, mbar_wait(&full[stage], phase, 300 + stage));
          const uint32_t b16 = resident ? bres_it16 : a_ring16 + ((2u * A_BYTES) >> 4);
          wgmma_fence();
          issue_tap<BLOCK_N, KSTEPS, SPLIT, !PP>(dm, dc, a_ring16 + wg16, lo16, kHiStd, b16, kB16, kHiStd, ksteps);
          unit_issued(stage, -1);  // frees this smem stage once the MMAs above have read it
          a_ring16 += stage16;
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
            a_ring16 = ring16;
          }
        }
      }
      if (PP && pass_turn) named_bar_arrive(4 + (wg ^ 1), kEpiThreads);
      wgmma_wait<0>();
      wgmma_fence_regs(dm);
      if constexpr (SPLIT) wgmma_fence_regs(dc);
      if (lane == 0) {
        if (pend_a >= 0) mbar_arrive(&empty[pend_a]);
        if (pend_b >= 0) mbar_arrive(&emptyB[pend_b]);
      }
      pend_a = pend_b = -1;
      const float gain = a.rz_gain;
#pragma unroll
      for (int i = 0; i < BLOCK_N / 2; ++i) {
        if constexpr (SPLIT) dm[i] = fmaf(dm[i], gain, dc[i]);
        else dm[i] *= gain;
      }
    };
    // accumulator columns [c0, c0 + ncols) of this thread's fragment -> acc_s (columns relative to c0).  wgmma fragment: rows
    // 64*wg + 16*(warp&3) + lane/4 (+8), columns 8*j + 2*(lane&3) (+1); in both schedules accumulator row 64*wg + r holds wgmma row r
    const int fr = 64 * wg + 16 * q + (lane >> 2), fc = 2 * (lane & 3);
    auto dump = [&](int c0, int ncols) {
#pragma unroll
      for (int j = 0; j < ncols / 8; ++j) {
        const int jj = c0 / 8 + j;
        float* p0 = acc_s + fr * ACC_PITCH + 8 * j + fc;
        *reinterpret_cast<float2*>(p0) = make_float2(dm[4 * jj], dm[4 * jj + 1]);
        *reinterpret_cast<float2*>(p0 + 8 * ACC_PITCH) = make_float2(dm[4 * jj + 2], dm[4 * jj + 3]);
      }
    };
    constexpr int kGroups = BLOCK_N / OUT_GROUP_CH;
    auto dump_group = [&](int g) {  // (unrolled: the fragment registers are indexed with constants only)
#pragma unroll
      for (int gg = 0; gg < kGroups; ++gg)
        if (gg == g) dump(gg * OUT_GROUP_CH, OUT_GROUP_CH);
    };

    int cur_n0 = -1;
    uint32_t gcount = 0;
    uint32_t res_phase = 0;
    grid_dep_wait();  // residual / up-partial reads and the output stores must not pass the previous kernel(s)
    const float rscale = (EPI == 2 || EPI == 4) ? 1.0f : a.resid_scale;  // (the specialised kernels are selected for unit shortcuts only)
    // residual tile of (tile, group): two TMA boxes (hi, lo) with the output tile's geometry; OOB parts are zero-filled
    auto issue_residual = [&](int tile_i, int g) {
      const TileOrigin to = tile_origin<BLOCK_N>(a, tile_i);
      const int c0 = to.n0 + g * OUT_GROUP_CH;
      mbar_expect_tx(rfull_t, (uint32_t)(2 * a.rows_valid * OUT_ROW_BYTES));
      tma_load_5d(&a.tmR, rfull_t, res_t, c0, to.w0, to.h0, to.b0, 0);
      tma_load_5d(&a.tmR, rfull_t, res_t + OUT_PLANE_BYTES, c0, to.w0, to.h0, to.b0, 1);
    };
    // fused YOLOv5 decode (YOLO kernels): staging tile [128 rows][85] fp32 + per-row partial best scores + per-image NMS histogram
    float* y_stage = reinterpret_cast<float*>(out_stage0);
    float* y_part = y_stage + kTileM * 85;
    uint32_t* hist_s = reinterpret_cast<uint32_t*>(out_stage0 + kYoloStageBytes);
    int cur_img = -1;
    auto flush_hist = [&](int img) {  // all epilogue threads: add the CTA's counts of image `img` to the workspace histogram
      named_bar_sync(1, EPI_THREADS);
      if (img >= 0 && a.y_hist != nullptr) {
        unsigned int* gh = a.y_hist + (size_t)img * kNmsBins;
        for (int i = tid_e; i < kNmsBins; i += EPI_THREADS) {
          const uint32_t c = hist_s[i];
          if (c) {
            atomicAdd(&gh[i], c);
            hist_s[i] = 0;
          }
        }
      }
      named_bar_sync(1, EPI_THREADS);
    };
    float* y_bias = reinterpret_cast<float*>(out_stage0 + kYoloStageBytes + kNmsBins * 4);  // [anchor][128]; -inf in the padding columns: sigmoid = 0, never a candidate
    if constexpr (YOLO) {
      for (int i = tid_e; i < kNmsBins; i += EPI_THREADS) hist_s[i] = 0;
      for (int i = tid_e; i < a.tiles_n * BLOCK_N; i += EPI_THREADS)
        y_bias[i] = ((i & (BLOCK_N - 1)) < a.y_no && i < a.bias_len) ? a.bias[i] : -CUDART_INF_F;
    }
    // this thread's tiles: all of the CTA's, or (ping-pong) every other one, starting with the warpgroup's index
    const int my_begin = PP ? t_begin + wg * t_step : t_begin;
    const int my_step = PP ? 2 * t_step : t_step;
    if (resid_tma && tid_e == 0 && my_begin < t_end) issue_residual(my_begin, 0);
    if (a.b_resident && t_begin < t_end) mbar_wait(bfull, 0, 250);
    // per-thread pixel coordinates are needed only by the operands read with per-thread loads (up-partial, non-TMA residual) and by the
    // fused decode; the plain path knows its tile through the TMA store coordinates alone
    const bool need_rows = EPI != 0 ? false : (YOLO || a.up != nullptr || (a.resid != nullptr && !resid_tma));
    for (int tile = (dbg & 16) ? t_end : my_begin, kt = PP ? wg : 0; tile < t_end; tile += my_step, kt += PP ? 2 : 1) {
      const TileOrigin to = tile_origin<BLOCK_N>(a, tile);
      const int w0 = to.w0, h0 = to.h0, b0 = to.b0, n0 = to.n0;
      const int ow = w0 + tw, oh = h0 + th, ob = b0 + nb;
      const bool valid = need_rows && (row < a.rows_valid) && (ow < a.Wo) && (oh < a.Ho) && (ob < a.Bn);

      {
        const long long pt0 = prof_on ? clock64() : 0;
        if constexpr (PP) {
          // the producer fills the ring in the CTA's tile order: this tile (the CTA's kt-th) starts at ring position kt * k_iters
          const int pos = kt * k_iters;
          stage = pos % STAGES;
          phase = (uint32_t)(pos / STAGES) & 1u;
          a_ring16 = ring16 + (uint32_t)stage * stage16;
          if (kt > 0) named_bar_sync(4 + wg, kEpiThreads);  // wait for the turn: the other warpgroup has issued the previous tile
        }
        mainloop(tile + t_step < t_end);
        if (prof_on) prof_acc[0] += clock64() - pt0;  // MMA main loop (including the waits for operands and, ping-pong, for the turn)
      }

      if (!YOLO && n0 != cur_n0) {
        named_bar_sync(ebar, EPI_THREADS);
        for (int i = tid_e; i < BLOCK_N; i += EPI_THREADS) {
          float bv = (n0 + i < a.bias_len) ? a.bias[n0 + i] : 0.0f;
          bias_t[i] = bv;
        }
        named_bar_sync(ebar, EPI_THREADS);
        cur_n0 = n0;
      }
      const float* up_row = nullptr;
      if (EPI == 0 && a.up != nullptr && valid)
        up_row = a.up + ((size_t)((size_t)ob * a.up_H + (oh >> 1)) * a.up_W + (ow >> 1)) * a.up_pitch + n0;
      const __half* res_row = nullptr;
      if (EPI == 0 && a.resid != nullptr && valid) res_row = a.resid + ((size_t)((size_t)ob * a.Ho + oh) * a.Wo + ow) * a.resid_pitch + n0;

      if constexpr (YOLO) {
        // ---- conv -> sigmoid -> box decode -> z rows + NMS histogram + per-row best score, straight from the accumulator
        // (replaces the fp32 raw tensor round trip + cvb_yolo_decode: yolov5_detect.py:42-55; same arithmetic, bit-identical z).
        // n-tile nt == anchor; accumulator column o < y_no is output o of that anchor; thread == pixel row of the tile.  The level is
        // seen as ONE row of ny*nx pixels (the planner flattens the 1x1 conv), so a tile's 128 pixels are 128 consecutive z rows.
        // Two decode groups (accumulator rows 0-63 / 64-127 = the two warpgroups) with their own staging half, barrier and TMA bulk
        // store, so one group's copy-out overlaps the other's conversion; in a group, two warps per row (`part`), three of the six
        // 16-column chunks each.
        if (b0 != cur_img) {  // (NB == 1 in this mode: one image per tile; b0 is uniform over the CTA)
          flush_hist(cur_img);
          cur_img = b0;
        }
        const int an = n0 / BLOCK_N, no = a.y_no;
        const float conf = a.y_conf;
        const float* bias_a = y_bias + an * BLOCK_N;
        const int grp = wg;                                      // rows 64 * grp .. + 63
        const int part = half;                                   // 0..1
        constexpr int GT = EPI_THREADS / 2;                      // threads per group
        const int gtid = q * 32 + lane;                          // thread index inside the group
        const int npix = a.Wo;                                   // pixels of the level (flattened)
        const int py = (int)__umulhi((uint32_t)ow, a.y_nx_magic), px = ow - py * a.y_nx;  // ow = flat pixel index
        const size_t lvl_row0 = (size_t)b0 * (size_t)a.y_zrows + (size_t)a.y_zoff + (size_t)an * npix;  // z row of the level's pixel 0
        // the group's accumulator rows were last read before the group barrier that ended its previous conversion
        dump(0, 96);
        // the group's staging half was last read by the bulk store its thread 0 issued for the previous tile
        long long pt0 = prof_on ? clock64() : 0;
        if (gtid == 0) tma_store_wait_read0();
        named_bar_sync(2 + grp, GT);
        if (prof_on) {
          const long long t = clock64();
          prof_acc[1] += t - pt0;  // waiting for the staging half (previous bulk store + group barrier)
          pt0 = t;
        }
        const float* arow = acc_s + row * ACC_PITCH;
        // objectness of this thread's row; 0 for rows outside the level, so that none of their scores passes the threshold
        const float obj = valid ? sigmoid_fast(arow[4] + bias_a[4]) : 0.0f;
        float rbest = 0.0f;
        float* srow = y_stage + row * 85;
        const uint32_t hist_s32 = smem_u32(hist_s);
        const bool any_live = __any_sync(0xffffffffu, obj > conf);  // background-only warps skip the score pass
        const bool multi = a.y_multi != 0 && !(dbg & 32);
#pragma unroll 1
        for (int cg = 0; cg < 3; ++cg) {  // this warp's 16-column chunks: part, part + 2, part + 4 (columns >= 96 are padding)
          const int col = (part + 2 * cg) * 16;
          if (col >= no || (dbg & 4)) break;
          float yv[16];
#pragma unroll
          for (int j = 0; j < 4; ++j) {  // 16 independent sigmoids: the MUFU pipe stays busy (bias is -inf beyond the anchor's outputs: y = 0)
            const float4 v4 = *reinterpret_cast<const float4*>(arow + col + 4 * j);
            yv[4 * j + 0] = sigmoid_fast(v4.x + bias_a[col + 4 * j + 0]);
            yv[4 * j + 1] = sigmoid_fast(v4.y + bias_a[col + 4 * j + 1]);
            yv[4 * j + 2] = sigmoid_fast(v4.z + bias_a[col + 4 * j + 2]);
            yv[4 * j + 3] = sigmoid_fast(v4.w + bias_a[col + 4 * j + 3]);
          }
          int j0 = 0;
          if (col == 0) {  // (warp-uniform) box columns
            srow[0] = yolo_xy(yv[0], (float)px, a.y_stride);
            srow[1] = yolo_xy(yv[1], (float)py, a.y_stride);
            srow[2] = yolo_wh(yv[2], a.y_anchor[an * 2]);
            srow[3] = yolo_wh(yv[3], a.y_anchor[an * 2 + 1]);
            srow[4] = yv[4];
            yv[0] = yv[1] = yv[2] = yv[3] = yv[4] = 0.0f;  // not class scores
            j0 = 5;
          }
          if (col + 16 <= no) {
#pragma unroll
            for (int j = 0; j < 16; ++j)
              if (j >= j0) srow[col + j] = yv[j];
          } else {
#pragma unroll
            for (int j = 0; j < 16; ++j)
              if (j >= j0 && col + j < no) srow[col + j] = yv[j];
          }
          if (any_live) {
            // y = 0 in the padding columns and obj = 0 in rows outside the level, so `sc > conf` alone decides; the histogram update
            // sits behind a warp vote (a uniform branch): background pixels cost four instructions per score
#pragma unroll
            for (int j = 0; j < 16; ++j) {
              const float sc = yolo_score(yv[j], obj);
              const bool pass = sc > conf;
              rbest = fmaxf(rbest, sc);
              if (multi && __any_sync(0xffffffffu, pass)) hist_inc_if(hist_s32, sc, pass);
            }
          }
        }
        y_part[part * kTileM + row] = rbest;
        fence_proxy_async_smem();  // generic-proxy smem writes -> visible to the bulk-copy engine (async proxy)
        if (prof_on) {
          const long long t = clock64();
          prof_acc[2] += t - pt0;  // conversion
          pt0 = t;
        }
        named_bar_sync(2 + grp, GT);
        if (prof_on) {
          const long long t = clock64();
          prof_acc[3] += t - pt0;  // group barrier after the conversion
          pt0 = t;
        }
        {
          // the group's valid tile rows [r0, r1) are consecutive z rows: one bulk copy
          const int r0 = grp * 64;
          const int r1 = min(min(r0 + 64, a.rows_valid), npix - w0);
          if (r1 > r0 && !(dbg & 64)) {
            float* gdst = a.yz + (lvl_row0 + (size_t)(w0 + r0)) * (size_t)no;
            const float* ssrc = y_stage + (size_t)r0 * 85;
            const int nfl = (r1 - r0) * no;
            if (no == 85 && (reinterpret_cast<uintptr_t>(gdst) & 15) == 0 && (nfl & 3) == 0 && !(dbg & 128)) {
              if (gtid == 0) {
                bulk_store_1d(gdst, ssrc, (uint32_t)nfl * 4u);
                tma_store_commit();
              }
            } else if (no == 85) {  // generic paths (odd geometry / fewer classes): staged rows have pitch 85, z rows pitch `no`
              for (int i = gtid; i < nfl; i += GT) gdst[i] = ssrc[i];
            } else {
              for (int i = gtid; i < nfl; i += GT) gdst[i] = ssrc[(i / no) * 85 + (i % no)];
            }
          }
          if (a.y_rowmax != nullptr && part == 0 && valid) {
            float rm = fmaxf(y_part[row], y_part[kTileM + row]);
            if (!(rm > conf)) rm = 0.0f;
            a.y_rowmax[lvl_row0 + (size_t)ow] = rm;
            if (!a.y_multi && rm > conf) atomicAdd(&hist_s[nms_score_bin(rm)], 1u);
          }
        }
        if (prof_on) prof_acc[4] += clock64() - pt0;  // copy-out issue + rowmax
        continue;
      }
#pragma unroll 1
      for (int g = 0; g < kGroups; ++g) {
        const int col0 = g * OUT_GROUP_CH + half * CW;
        const bool ch_ok = (n0 + col0 + CW <= a.cout);
        const bool has_up = EPI != 0 ? false : ((up_row != nullptr) && ch_ok);
        const bool has_res = (EPI == 1 || EPI == 3) ? false : (resid_tma ? true : ((res_row != nullptr) && ch_ok));
        // the thread's CW columns are processed in sub-chunks of SUB columns (SUB < CW only for the small-N kernels that must
        // stay within the two-CTAs-per-SM register budget).  Epilogue operands that do not depend on the accumulator are
        // requested first, so their latency hides behind the accumulator staging / barrier below
        float4 upv[SUB / 4];
        uint4 rhv[SUB / 8], rlv[SUB / 8];
        auto load_extras = [&](int sc) {
          const int col = col0 + sc * SUB;
          if (has_up) {
            const float4* p = reinterpret_cast<const float4*>(up_row + col);
#pragma unroll
            for (int j = 0; j < SUB / 4; ++j) upv[j] = __ldg(p + j);
          }
          if (has_res && !resid_tma) {
            const uint4* ph = reinterpret_cast<const uint4*>(res_row + col);
            const uint4* pl = reinterpret_cast<const uint4*>(res_row + a.resid_plane + col);
#pragma unroll
            for (int j = 0; j < SUB / 8; ++j) {
              rhv[j] = __ldg(ph + j);
              rlv[j] = __ldg(pl + j);
            }
          }
        };
        load_extras(0);
        if constexpr (!OUT_F32) {
          if (resid_tma) {
            mbar_wait(rfull_t, res_phase, 500);
            res_phase ^= 1;
          }
        }
        // the accumulator tile was last read before the barrier that ended the previous group's conversion
        dump_group(g);
        // the staging tile written now was last read by the TMA store issued out_bufs groups ago
        long long pt0 = prof_on ? clock64() : 0;
        if (tid_e == 0) {
          if (a.out_bufs == 2) tma_store_wait_read1();
          else tma_store_wait_read0();
        }
        named_bar_sync(ebar, EPI_THREADS);
        if (prof_on) {
          const long long t = clock64();
          prof_acc[1] += t - pt0;  // staging tile free (TMA store read + barrier)
          pt0 = t;
        }
        uint8_t* out_stage = out_stage0 + (gcount & (a.out_bufs - 1)) * G.out_buf_bytes + (PP ? wg * OUT_TILE_BYTES : 0);
        ++gcount;
#pragma unroll
        for (int sc = 0; sc < CW / SUB; ++sc) {
          if (dbg & 4) break;  // diagnostics: no accumulator reads / math / staging
          const int col = col0 + sc * SUB;
          if (sc > 0) load_extras(sc);
          if constexpr (!OUT_F32) {
            if (resid_tma) {  // same swizzled chunk addressing as the output staging tile below
              const uint8_t* rh = res_t + row * OUT_ROW_BYTES;
#pragma unroll
              for (int j = 0; j < SUB / 8; ++j) {
                const int cj = half * (CW / 8) + sc * (SUB / 8) + j;
                int chunk;
                if constexpr (OUT_GROUP_CH == 64) chunk = cj ^ (row & 7);
                else chunk = cj ^ ((row >> 1) & 3);
                rhv[j] = *reinterpret_cast<const uint4*>(rh + (chunk << 4));
                rlv[j] = *reinterpret_cast<const uint4*>(rh + OUT_PLANE_BYTES + (chunk << 4));
              }
            }
          }
          float f[SUB];
          {
            const float* ap = acc_t + row * ACC_PITCH + (col - g * OUT_GROUP_CH);
#pragma unroll
            for (int j = 0; j < SUB / 4; ++j) {
              const float4 v4 = *reinterpret_cast<const float4*>(ap + 4 * j);
              f[4 * j] = v4.x;
              f[4 * j + 1] = v4.y;
              f[4 * j + 2] = v4.z;
              f[4 * j + 3] = v4.w;
            }
          }
          float bv[SUB];  // bias of this thread's columns: 16-byte shared-memory loads
#pragma unroll
          for (int j = 0; j < SUB / 4; ++j) {
            const float4 b4 = *reinterpret_cast<const float4*>(bias_t + col + 4 * j);
            bv[4 * j] = b4.x;
            bv[4 * j + 1] = b4.y;
            bv[4 * j + 2] = b4.z;
            bv[4 * j + 3] = b4.w;
          }
          if (dbg & 256) continue;  // diagnostics: accumulator reads only
          if (has_up) {
#pragma unroll
            for (int j = 0; j < SUB / 4; ++j) {
              f[4 * j + 0] += upv[j].x;
              f[4 * j + 1] += upv[j].y;
              f[4 * j + 2] += upv[j].z;
              f[4 * j + 3] += upv[j].w;
            }
          }
          float rsum[SUB];  // residual (hi + lo) of this thread's pixel, 0 when absent
#pragma unroll
          for (int j = 0; j < SUB; ++j) rsum[j] = 0.0f;
          if (has_res) {
#pragma unroll
            for (int j = 0; j < SUB / 8; ++j) {
              const __half2* h2 = reinterpret_cast<const __half2*>(&rhv[j]);
              const __half2* l2 = reinterpret_cast<const __half2*>(&rlv[j]);
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const float2 hf = __half22float2(h2[e]);
                const float2 lf = __half22float2(l2[e]);
                rsum[8 * j + 2 * e + 0] = (hf.x + lf.x) * rscale;
                rsum[8 * j + 2 * e + 1] = (hf.y + lf.y) * rscale;
              }
            }
          }
          const bool rf = EPI == 4 ? true : (EPI != 0 ? false : (a.resid_first != 0));
          if (act_mode == CVB_ACT_SILU) {
#pragma unroll
            for (int j = 0; j < SUB; ++j) {
              const float t = f[j] + bv[j];
              f[j] = rf ? silu_fast(t + rsum[j]) : silu_fast(t) + rsum[j];
            }
          } else if (act_mode == CVB_ACT_RELU) {
#pragma unroll
            for (int j = 0; j < SUB; ++j) {
              const float t = f[j] + bv[j];
              f[j] = rf ? fmaxf(t + rsum[j], 0.0f) : fmaxf(t, 0.0f) + rsum[j];
            }
          } else {
#pragma unroll
            for (int j = 0; j < SUB; ++j) f[j] = f[j] + bv[j] + rsum[j];
          }
          if (dbg & 512) {  // diagnostics: no conversion / staging stores (the results stay live through a dummy dependency)
            float acc_d = 0.0f;
#pragma unroll
            for (int j = 0; j < SUB; ++j) acc_d += f[j];
            if (acc_d == 123.456f) bias_s[0] = acc_d;
            continue;
          }
          if constexpr (OUT_F32) {
            // row = 32 fp32 = 128 B = 8 chunks of 16 B, 128B swizzle: chunk ^= row & 7; this warp owns chunks half*4 .. +3
            uint8_t* rowp = out_stage + row * 128;
#pragma unroll
            for (int j = 0; j < SUB / 4; ++j) {
              const uint4 o = make_uint4(__float_as_uint(f[4 * j]), __float_as_uint(f[4 * j + 1]), __float_as_uint(f[4 * j + 2]),
                                         __float_as_uint(f[4 * j + 3]));
              *reinterpret_cast<uint4*>(rowp + (((half * (CW / 4) + sc * (SUB / 4) + j) ^ (row & 7)) << 4)) = o;
            }
          } else {
            uint8_t* rowh = out_stage + row * OUT_ROW_BYTES;
            uint8_t* rowl = rowh + OUT_PLANE_BYTES;
#pragma unroll
            for (int j = 0; j < SUB / 8; ++j) {
              uint32_t hq[4], lq[4];
#pragma unroll
              for (int e = 0; e < 4; ++e) split_pair(f[8 * j + 2 * e], f[8 * j + 2 * e + 1], hq[e], lq[e]);
              const int cj = half * (CW / 8) + sc * (SUB / 8) + j;  // 16-byte chunk (8 channels) inside the staged row
              int chunk;
              if constexpr (OUT_GROUP_CH == 64) chunk = cj ^ (row & 7);   // 128B swizzle
              else chunk = cj ^ ((row >> 1) & 3);                         // 64B swizzle
              *reinterpret_cast<uint4*>(rowh + (chunk << 4)) = make_uint4(hq[0], hq[1], hq[2], hq[3]);
              *reinterpret_cast<uint4*>(rowl + (chunk << 4)) = make_uint4(lq[0], lq[1], lq[2], lq[3]);
            }
          }
        }
        fence_proxy_async_smem();  // generic-proxy smem writes -> visible to the TMA (async proxy)
        if (prof_on) {
          const long long t = clock64();
          prof_acc[2] += t - pt0;  // accumulator reads + conversion + staging
          pt0 = t;
        }
        named_bar_sync(ebar, EPI_THREADS);
        if (prof_on) {
          const long long t = clock64();
          prof_acc[3] += t - pt0;  // barrier after the conversion
          pt0 = t;
        }
        if (tid_e == 0) {
          const int c0 = n0 + g * OUT_GROUP_CH;
          if (c0 < a.cout && !(dbg & 1)) {
            tma_store_5d(&a.tmO, out_stage, c0, w0, h0, b0, 0);
            if constexpr (!OUT_F32) tma_store_5d(&a.tmO, out_stage + OUT_PLANE_BYTES, c0, w0, h0, b0, 1);
          }
          tma_store_commit();
          if (resid_tma) {  // every epilogue thread has consumed the residual tile (barrier above): fetch the next one
            if (g + 1 < kGroups) issue_residual(tile, g + 1);
            else if (tile + my_step < t_end) issue_residual(tile + my_step, 0);
          }
        }
        if (prof_on) prof_acc[4] += clock64() - pt0;  // store issue
      }
    }
    if constexpr (YOLO) {
      flush_hist(cur_img);
      if (q == 0 && lane == 0) tma_store_wait_all0();  // thread 0 of each decode group: its bulk stores
    }
    if (tid_e == 0) tma_store_wait_all0();
    if (prof_on && tid_e == 0) {  // epilogue: total cycles, MMA main loop, staging waits, conversion, barrier, store issue, and (classic
                                  // loader) the main loop's waits on the ring's full barriers
      long long* pr = a.prof + ((size_t)(PP ? wg : 0) * gridDim.x + blockIdx.x) * 16;  // ping-pong: one counter row per warpgroup
      pr[8] = clock64() - prof_t0;
      pr[9] = prof_acc[0];
      for (int i = 1; i < 6; ++i) pr[9 + i] = prof_acc[i];
    }
  }
}

// ---------------------------------------------------------------------------------------------- host
template <int BN, int BK, bool PP, int CTAS = 1>
static const void* kernel_epi(bool f32, int epi) {
  if (f32) return reinterpret_cast<const void*>(&conv_tc_kernel<BN, BK, true, false, 0, PP, CTAS>);
  switch (epi) {
    case 1: return reinterpret_cast<const void*>(&conv_tc_kernel<BN, BK, false, false, 1, PP, CTAS>);
    case 2: return reinterpret_cast<const void*>(&conv_tc_kernel<BN, BK, false, false, 2, PP, CTAS>);
    case 3: return reinterpret_cast<const void*>(&conv_tc_kernel<BN, BK, false, false, 3, PP, CTAS>);
    case 4: return reinterpret_cast<const void*>(&conv_tc_kernel<BN, BK, false, false, 4, PP, CTAS>);
    default: return reinterpret_cast<const void*>(&conv_tc_kernel<BN, BK, false, false, 0, PP, CTAS>);
  }
}

// The cooperative block_n <= 64 kernels.  ctas == 1: the one-CTA register bound, instantiated for the epilogues a one-CTA-per-SM
// cooperative plan gets in auto mode (no residual tile: the narrow layers with a residual run ping-pong); the residual epilogues keep the
// two-CTA bound.
template <int BN, int BK>
static const void* kernel_narrow(bool f32, int epi, int ctas) {
  if (ctas == 1) {
    if (f32) return reinterpret_cast<const void*>(&conv_tc_kernel<BN, BK, true, false, 0, false, 1>);
    if (epi == 0) return reinterpret_cast<const void*>(&conv_tc_kernel<BN, BK, false, false, 0, false, 1>);
    if (epi == 1) return reinterpret_cast<const void*>(&conv_tc_kernel<BN, BK, false, false, 1, false, 1>);
    if (epi == 3) return reinterpret_cast<const void*>(&conv_tc_kernel<BN, BK, false, false, 3, false, 1>);
  }
  return kernel_epi<BN, BK, false, 2>(f32, epi);
}

// The kernel instantiation, or nullptr.  pp: the ping-pong schedule, instantiated for block_n <= 128 (at 256 its generic and residual
// epilogues spill more than the cooperative kernel's).  ctas: CTAs per SM of the plan (selects the register bound of the cooperative
// narrow kernels).
static const void* lookup_kernel(int bn, int bk, bool f32, bool yolo = false, int epi = 0, bool pp = false, int ctas = 1) {
  if (yolo) {  // fused-decode epilogue: one anchor per 128-wide n-tile
    if (pp) return nullptr;
    if (bn == 128 && bk == 32) return reinterpret_cast<const void*>(&conv_tc_kernel<128, 32, true, true>);
    if (bn == 128 && bk == 64) return reinterpret_cast<const void*>(&conv_tc_kernel<128, 64, true, true>);
    return nullptr;
  }
#define CVB_CASE(BN, BK) \
  if (bn == BN && bk == BK) return kernel_epi<BN, BK, false>(f32, epi);
#define CVB_CASE_PP(BN, BK) \
  if (bn == BN && bk == BK) return pp ? kernel_epi<BN, BK, true>(f32, epi) : kernel_epi<BN, BK, false>(f32, epi);
#define CVB_CASE_NARROW(BN, BK) \
  if (bn == BN && bk == BK) return pp ? kernel_epi<BN, BK, true>(f32, epi) : kernel_narrow<BN, BK>(f32, epi, ctas);
  CVB_CASE_NARROW(32, 16) CVB_CASE_NARROW(32, 32) CVB_CASE_NARROW(32, 64)
  CVB_CASE_NARROW(64, 16) CVB_CASE_NARROW(64, 32) CVB_CASE_NARROW(64, 64)
  CVB_CASE_PP(128, 16) CVB_CASE_PP(128, 32) CVB_CASE_PP(128, 64)
  if (pp) return nullptr;
  CVB_CASE(256, 16) CVB_CASE(256, 32) CVB_CASE(256, 64)
#undef CVB_CASE
#undef CVB_CASE_PP
#undef CVB_CASE_NARROW
  return nullptr;
}

// A CTA's dynamic shared memory: `stages` ring slots of `slot` bytes, the weight region (resident slab or halo weight ring), the output
// staging tiles (fused decode: staging tile, NMS histogram and bias), the residual tile, the accumulator tile, the bias and the
// mbarriers.  Every plan is sized with it; the kernel chains the same regions in the same order (see its prologue).
static SmemLayout smem_layout(const ConvGeom& g, int stages, int slot, int weight_bytes, int out_bufs, bool resid_tma, bool yolo) {
  SmemLayout l;
  l.slot = slot;
  l.weights = stages * slot;
  l.out = l.weights + weight_bytes;
  l.resid = l.out + (yolo ? kYoloStageBytes + kNmsBins * 4 + kYoloBiasBytes : out_bufs * g.out_buf_bytes);
  l.acc = l.resid + (resid_tma ? g.out_buf_bytes : 0);
  l.bias = l.acc + g.acc_bytes;
  l.bars = l.bias + g.bias_bytes;
  l.total = l.bars + kBarBytes;
  return l;
}

// ring slots that fit in `budget` next to the other regions of l0 (a layout of 0 stages); 0 or less: no fit
static int stages_fitting(int budget, const SmemLayout& l0) { return (budget - l0.total) / l0.slot; }

}  // namespace cvb

struct CvbConvPlan {
  cvb::ConvKArgs args;
  const void* fn;
  int grid;
  int smem;
  int threads;
  int schedule;  // CVB_SCHED_COOPERATIVE or CVB_SCHED_PINGPONG
  int epi;       // compile-time epilogue specialisation of fn (0 = generic, see fill_epilogue)
};

namespace cvb {

static CUtensorMapSwizzle swizzle_for_bytes(int bytes) {
  return bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : (bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
}

// 5-D (C, W, H, B, plane) tensor map: extents, byte strides of a W / H / B / plane step, and the box
static int encode_5d(CUtensorMap* m, CUtensorMapDataType dt, const void* base, int C, int W, int H, int B, int planes, long long s_w,
                     long long s_h, long long s_b, long long s_plane, const int (&box)[5], CUtensorMapSwizzle swz) {
  const cuuint64_t dims[5] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B, (cuuint64_t)planes};
  const cuuint64_t str[4] = {(cuuint64_t)s_w, (cuuint64_t)s_h, (cuuint64_t)s_b, (cuuint64_t)s_plane};
  const cuuint32_t bx[5] = {(cuuint32_t)box[0], (cuuint32_t)box[1], (cuuint32_t)box[2], (cuuint32_t)box[3], (cuuint32_t)box[4]};
  return encode_map(m, dt, 5, base, dims, str, bx, swz);
}

// Pick the output pixel box (TW x TH x NB <= rows: the tile's accumulator rows) that wastes the fewest accumulator rows.
static void choose_box(int B, int H, int W, int rows, int* TW, int* TH, int* NB) {
  double best = -1.0;
  int bw = 1, bh = 1, bb = 1;
  for (int tw = 1; tw <= rows; ++tw) {
    if (tw > W && tw != 1) break;
    if (!(tw == W || (tw & (tw - 1)) == 0)) continue;  // powers of two, or the full row
    for (int th = 1; th * tw <= rows; ++th) {
      if (th > H) break;
      int nb = rows / (tw * th);
      if (nb > B) nb = B;
      if (nb < 1) nb = 1;
      // keep all box dims <= 256 (TMA limit) -- implied by <= 128
      const long long tiles = (long long)ceil_div(W, tw) * ceil_div(H, th) * ceil_div(B, nb);
      const double util = (double)B * H * W / ((double)tiles * rows);
      const double score = util + 1e-4 * tw / 128.0;  // tie-break: longer contiguous rows
      if (score > best) {
        best = score;
        bw = tw;
        bh = th;
        bb = nb;
      }
    }
  }
  *TW = bw;
  *TH = bh;
  *NB = bb;
}

// A/B knobs read once per process
static bool two_ctas_on() {
  static const bool on = [] {
    const char* e = getenv("CVB_CTAS_PER_SM");  // A/B knob: 1 = always one CTA per SM
    return !(e && atoi(e) == 1);
  }();
  return on;
}
static bool resid_tma_on() {
  static const bool on = [] {
    const char* e = getenv("CVB_RESID_TMA");  // A/B knob: 0 = per-thread residual loads
    return !(e && atoi(e) == 0);
  }();
  return on;
}

// The validated descriptor (the fused-decode level flattened to one row) and the GEMM view of the layer.
struct ConvProblem {
  CvbConvDesc d;
  int yolo_nx;  // fused decode: width of the level
  int win;      // >0: K chunk of a filter row = `win` horizontally adjacent input pixels (see cvb200.h)
  int cin;      // K per tap as seen by the GEMM
  int cout, Ho, Wo, n_taps;
  bool yolo, f32, has_resid;
};

// the K chunk that divides cin best
static int full_bk(int cin) { return (cin % 64 == 0) ? 64 : (cin % 32 == 0 ? 32 : 16); }

// the CTA's n-tile can stay the same along its stride over the tiles, so its weights may stay resident
static bool can_pin(int cout, int bn) { return ceil_div(cout, bn) == 1 || ceil_div(cout, bn) == 2 || ceil_div(cout, bn) == 4; }

static int validate_desc(const CvbConvDesc& desc, ConvProblem* P) {
  P->d = desc;
  CvbConvDesc* d = &P->d;
  P->yolo = d->out_kind == CVB_OUT_YOLO;
  P->yolo_nx = 0;
  if (P->yolo) {
    // fused decode: a 1x1 / stride 1 conv does not care about the image geometry, so the level is planned as ONE row of H * W pixels.
    // A tile is then 128 consecutive pixels = 128 consecutive z rows (one contiguous 43 KB store) and no accumulator row is wasted
    // on partial boxes (80x80: 50 full tiles per image and anchor).
    CVB_REQUIRE(d->in.H >= 1 && d->in.W >= 1 && d->in.H == d->out.H && d->in.W == d->out.W && (long long)d->in.H * d->in.W < (1 << 24),
                "conv(yolo): bad level geometry");
    P->yolo_nx = d->in.W;
    d->in.W = d->out.W = d->in.H * d->in.W;
    d->in.H = d->out.H = 1;
  }
  const CvbView& in = d->in;
  const CvbView& out = d->out;
  CVB_REQUIRE(in.base && (out.base || P->yolo) && d->weights && d->bias, "conv: null tensor pointer");
  CVB_REQUIRE(d->kh >= 1 && d->kw >= 1 && (d->w_window > 0 ? d->kh : d->kh * d->kw) <= kMaxTaps,
              "conv: kernel %dx%d unsupported (max %d taps)", d->kh, d->kw, kMaxTaps);
  CVB_REQUIRE(d->stride == 1 || d->stride == 2, "conv: stride %d unsupported", d->stride);
  CVB_REQUIRE(d->dilation >= 1, "conv: bad dilation");
  const int win = d->w_window;
  if (win > 0) {
    CVB_REQUIRE(d->stride == 1 && d->dilation == 1 && d->kw <= win && d->pad >= 0 && d->pad < d->kh,
                "conv: w_window needs a stride-1 convolution with kw <= w_window (filter row ky reads input row h + ky - pad)");
    CVB_REQUIRE(in.c_pitch == in.C && (win * in.C == 64 || win * in.C == 32), "conv: w_window needs contiguous pixels and window*C in {32,64}");
    CVB_REQUIRE(in.W > win - 1, "conv: padded input too narrow");
  }
  const int cin = win > 0 ? win * in.C : in.C;
  if (P->yolo) {
    CVB_REQUIRE(d->yolo != nullptr && d->yolo->z != nullptr, "conv: out_kind CVB_OUT_YOLO needs CvbConvDesc.yolo with a z pointer");
    CVB_REQUIRE(d->yolo->na >= 1 && d->yolo->na <= 4 && d->yolo->no >= 6 && d->yolo->no <= 85, "conv(yolo): na <= 4 and 6 <= no <= 85 supported");
    CVB_REQUIRE(d->kh == 1 && d->kw == 1 && d->stride == 1 && d->pad == 0 && win == 0, "conv(yolo): the detect conv is 1x1 / stride 1");
    CVB_REQUIRE(out.C == d->yolo->na * 128 && d->cout_pad == out.C, "conv(yolo): weights must be packed one anchor per 128-wide n-tile (C = na*128)");
    CVB_REQUIRE(!d->residual.base && !d->up_partial.base && d->act == CVB_ACT_NONE, "conv(yolo): no residual / partial / activation");
    CVB_REQUIRE(is_aligned(d->yolo->z, 4), "conv(yolo): z must be 4-byte aligned");
    if (int rc = check_level_rows("conv(yolo)", d->yolo->z_off, (long long)d->yolo->na * in.H * in.W, d->yolo->z_rows)) return rc;
  }
  const int cout = out.C;
  CVB_REQUIRE(cin % 16 == 0, "conv: cin=%d must be a multiple of 16", cin);
  CVB_REQUIRE(in.c_pitch % 8 == 0 && (P->yolo || out.c_pitch % 8 == 0), "conv: channel pitch must be a multiple of 8");
  CVB_REQUIRE(is_aligned(in.base, 16) && (P->yolo || is_aligned(out.base, 16)) && is_aligned(d->weights, 16),
              "conv: pointers must be 16-byte aligned");
  // window mode: the caller fixes the output height (asymmetric vertical padding is expressed by `pad` = rows above; rows
  // below come from TMA zero fill), e.g. the 7x7/s2/p3 ResNet stem == 4 filter rows over the space-to-depth input, pad 2.
  const int Ho = win > 0 ? out.H : (in.H + 2 * d->pad - d->dilation * (d->kh - 1) - 1) / d->stride + 1;
  const int Wo = win > 0 ? in.W - (win - 1) : (in.W + 2 * d->pad - d->dilation * (d->kw - 1) - 1) / d->stride + 1;
  CVB_REQUIRE(Ho == out.H && Wo == out.W && in.B == out.B, "conv: output view %dx%dx%d does not match computed %dx%dx%d", out.B, out.H,
              out.W, in.B, Ho, Wo);
  CVB_REQUIRE(d->cout_pad >= cout && d->cout_pad % 8 == 0, "conv: bad cout_pad");
  P->f32 = d->out_kind == CVB_OUT_F32 || P->yolo;
  if (P->f32) CVB_REQUIRE(out.c_pitch % 4 == 0, "conv: fp32 output pitch must be a multiple of 4");
  if (d->residual.base) {
    const CvbView& r = d->residual;
    CVB_REQUIRE(r.B == out.B && r.H == Ho && r.W == Wo && r.C == cout && r.c_pitch % 8 == 0 && cout % 32 == 0 &&
                    is_aligned(r.base, 16) && r.plane_stride % 16 == 0,
                "conv: residual view mismatch");
  }
  if (d->up_partial.base) {
    const CvbView& u = d->up_partial;
    CVB_REQUIRE(u.B == out.B && u.H == (Ho + 1) / 2 && u.W == (Wo + 1) / 2 && u.C == cout && u.c_pitch % 4 == 0 && cout % 32 == 0 &&
                    is_aligned(u.base, 16),
                "conv: up_partial view mismatch");
  }
  P->win = win;
  P->cin = cin;
  P->cout = cout;
  P->Ho = Ho;
  P->Wo = Wo;
  P->n_taps = win > 0 ? d->kh : d->kh * d->kw;
  P->has_resid = d->residual.base != nullptr;
  return CVB_OK;
}

static int choose_block(const ConvProblem& P, int* bn_out, int* bk_out) {
  const CvbConvDesc* d = &P.d;
  const int cin = P.cin, cout = P.cout;
  int bn = d->block_n;
  if (bn == 0) {
    bn = cout <= 32 ? 32 : (cout <= 64 ? 64 : 128);
    static const int split128 = [] {
      // 128-wide 1x1 layers with cin <= 128 and an up-sampled partial run as two pinned 64-wide n-tiles (one CTA per SM, ping-pong):
      // the partial needs the generic epilogue, which spills at block_n = 128 and not at 64 (0.26 vs 0.50 ms at 80x80, B = 64).
      // Without the partial, one 128-wide ping-pong tile measured between 2 % slower and 11 % faster than two 64-wide ones, 0.03 ms
      // less over the eight such layers of the YOLOv5-s step (DESIGN.md 6).  Both give bitwise-equal outputs.  CVB_SPLIT_N128=0 keeps
      // one 128-wide tile per CTA.
      const char* e = getenv("CVB_SPLIT_N128");
      return e ? atoi(e) : 1;
    }();
    if (split128 && !P.f32 && d->kh * d->kw == 1 && cout == 128 && cin <= 128 && cin % 64 == 0 && d->up_partial.base) bn = 64;
  }
  int bk = full_bk(cin);
  if (P.yolo) {
    bn = 128;  // one anchor per n-tile
    CVB_REQUIRE(cin % 32 == 0, "conv(yolo): cin must be a multiple of 32");
    bk = 32;   // the 64 KB NMS histogram + 44 KB staging tile leave room for three 32 KB stages
  } else {
    static const int bk_small = [] {
      const char* e = getenv("CVB_BK_SMALLN");  // A/B knob: K chunk of the block_n <= 64 kernels for 64-channel inputs (default: full)
      const int v = e ? atoi(e) : 0;
      return (v == 16 || v == 32 || v == 64) ? v : 0;
    }();
    // 64-channel inputs into narrow tiles (1x1 convs and the row-window stems) keep the full 64-wide K chunk.  Half-size chunks shrink
    // the ring stages so that more of these plans fit two CTAs per SM, but on the H100 the YOLOv5-s step measured 0.3 ms faster with
    // full chunks (14.06-14.12 vs 14.40-14.41 ms, DESIGN.md 6).  CVB_BK_SMALLN=32 restores the half-size chunks.
    if (bk_small && bn <= 64 && (cin == 64 || (cin == 128 && cout > 64)) && (d->kh * d->kw == 1 || P.win > 0)) bk = bk_small;
  }
  *bn_out = bn;
  *bk_out = bk;
  return CVB_OK;
}

// ---- filter taps: (input map, row offset, column offset) of every tap; stride 2 reads four "parity" maps
struct TapTable {
  int8_t map[kMaxTaps], dh[kMaxTaps], dw[kMaxTaps];
};

static int build_taps(const ConvProblem& P, TapTable* T) {
  const CvbConvDesc* d = &P.d;
  if (P.win > 0) {
    for (int ky = 0; ky < d->kh; ++ky) {
      T->map[ky] = 0;
      T->dh[ky] = (int8_t)(ky - d->pad);
      T->dw[ky] = 0;  // the physical tensor carries the left zero column: window of output w starts at padded column w
    }
    return CVB_OK;
  }
  for (int ky = 0; ky < d->kh; ++ky)
    for (int kx = 0; kx < d->kw; ++kx) {
      const int t = ky * d->kw + kx;
      const int qy = ky * d->dilation - d->pad, qx = kx * d->dilation - d->pad;
      CVB_REQUIRE(qy >= -127 && qy <= 127 && qx >= -127 && qx <= 127, "conv: tap offset %d/%d out of the supported range", qy, qx);
      if (d->stride == 1) {
        T->map[t] = 0;
        T->dh[t] = (int8_t)qy;
        T->dw[t] = (int8_t)qx;
      } else {
        const int py = ((qy % 2) + 2) % 2, px = ((qx % 2) + 2) % 2;
        T->map[t] = (int8_t)(py * 2 + px);
        T->dh[t] = (int8_t)((qy - py) / 2);
        T->dw[t] = (int8_t)((qx - px) / 2);
      }
    }
  return CVB_OK;
}

// ---- halo (copy / tap) mode: see ConvKArgs.  Geometry is fixed to 8 x 16 output pixels of one image per tile, so the 8-row groups of
// every tap view are 8 horizontally adjacent pixels and consecutive groups are one (halo) image row apart.
constexpr int kHaloTW = 8, kHaloTH = 16;

struct HaloCfg {
  int mode = 0, bk = 0, resident = 0, sa = 0, sb = 0, out_bufs = 1, resid_tma = 0, ctas = 1;
  int n_copies = 0, fused = 1;
  int cp_map[6], cp_dw[6], cp_dh[6], cp_ntaps[6], cp_boxw[6], cp_boxh[6];
  int cp_ny[6], cp_nx[6], cp_w0[6], cp_wy[6], cp_wx[6];  // taps of a copy as an ny x nx grid, weight tap = w0 + y*wy + x*wx
  uint32_t cp_bytes[6], cp_lo_off[6], slot = 0;
  int tap_w[kMaxTaps], tap_off[kMaxTaps];
  int map_boxw[4], map_boxh[4];
  int kskip = 0;
  double cost = 0.0;
};

// The halo plan of the layer if the cost model (or a request) picks the halo loader; bk: the classic loader's K chunk.
static bool plan_halo(const ConvProblem& P, const TapTable& T, int bn, int bk, HaloCfg* out) {
  const CvbConvDesc* d = &P.d;
  const int n_taps = P.n_taps, cin = P.cin, cout = P.cout, win = P.win;
  const bool pin = can_pin(cout, bn);
  auto f_mma = [](int n) { return n / 2 > 50 ? n / 2 : 50; };  // cost model: cycles of one M=128, K=16 MMA step (floor of 50)
  const int chain_all = n_taps * cin / 16;
  const bool pair_mode_est = chain_all <= 160 && bn <= 128 && (bn == 128 || n_taps > 1);
  const double kstep_clk = pair_mode_est ? f_mma(2 * bn) + f_mma(bn) : 3.0 * f_mma(bn);
  const double kFillBpc = 40.0;  // L2 -> shared memory fill bandwidth per SM and clock when every SM pulls (measured ~6300 B/clk per chip)
  const int halo_env = [] {
    const char* e = getenv("CVB_HALO");  // A/B knob: 0 = classic one-box-per-tap loads everywhere, 1 / 2 = force that halo mode where possible
    return e ? atoi(e) : -1;
  }();
  const int HTW = kHaloTW, HTH = kHaloTH;
  const int halo_req = d->halo != 0 ? d->halo : halo_env;  // per-plan request wins over the environment knob
  if (!(n_taps > 1 && d->dilation == 1 && halo_req != 0 && halo_req != -2 && d->halo != -1)) return false;
  // the halo loader pays off where two CTAs share an SM (BLOCK_N <= 64: the
  // second CTA's MMAs fill the tensor-pipe bubbles of the first); mode 1 (aligned copies) wins for 32-channel inputs, mode 2 above
  const int mode = halo_req == 1 ? 1 : (halo_req == 2 ? 2 : (cin <= 32 && win == 0 ? 1 : 2));
  // copies: mode 2 = one per input map (box covers every tap of the map); mode 1 = one per (map, column offset)
  HaloCfg h;
  h.mode = mode;
  int nc = 0;
  int n_ord = 0;
  for (int m = 0; m < 4; ++m) {
    int dwmin = 127, dwmax = -127, dhmin = 127, dhmax = -127, cnt = 0;
    for (int t = 0; t < n_taps; ++t)
      if (T.map[t] == m) {
        dwmin = T.dw[t] < dwmin ? T.dw[t] : dwmin;
        dwmax = T.dw[t] > dwmax ? T.dw[t] : dwmax;
        dhmin = T.dh[t] < dhmin ? T.dh[t] : dhmin;
        dhmax = T.dh[t] > dhmax ? T.dh[t] : dhmax;
        ++cnt;
      }
    h.map_boxw[m] = h.map_boxh[m] = 0;
    if (!cnt) continue;
    h.map_boxh[m] = HTH + (dhmax - dhmin);
    h.map_boxw[m] = mode == 2 ? HTW + (dwmax - dwmin) : HTW;
    const int n_groups = mode == 2 ? 1 : (dwmax - dwmin + 1);
    for (int gi = 0; gi < n_groups; ++gi) {
      const int gdw = dwmin + gi;
      int nt = 0;
      int dhs[kMaxTaps], dws[kMaxTaps], ndh = 0, ndw = 0;
      for (int t = 0; t < n_taps; ++t)
        if (T.map[t] == m && (mode == 2 || T.dw[t] == gdw)) {
          h.tap_w[n_ord] = t;
          h.tap_off[n_ord] = (T.dh[t] - dhmin) * h.map_boxw[m] + (mode == 2 ? T.dw[t] - dwmin : 0);
          ++n_ord;
          ++nt;
          bool seen = false;
          for (int i = 0; i < ndh; ++i) seen |= dhs[i] == T.dh[t];
          if (!seen) dhs[ndh++] = T.dh[t];
          seen = false;
          for (int i = 0; i < ndw; ++i) seen |= dws[i] == T.dw[t];
          if (!seen) dws[ndw++] = T.dw[t];
        }
      if (!nt) continue;
      if (nc >= 6) {
        nc = 7;
        break;
      }
      {
        // the kernel walks the taps of a copy as an ny x nx grid with affine view offsets / weight indices: verify that structure
        auto find = [&](int dh, int dw) {
          for (int t = 0; t < n_taps; ++t)
            if (T.map[t] == m && T.dh[t] == dh && T.dw[t] == dw) return t;
          return -1;
        };
        bool affine = ndh * ndw == nt;
        const int t00 = find(dhs[0], dws[0]);
        const int wy = ndh > 1 ? find(dhs[1], dws[0]) - t00 : 0, wx = ndw > 1 ? find(dhs[0], dws[1]) - t00 : 0;
        for (int y = 0; affine && y < ndh; ++y)
          for (int x = 0; affine && x < ndw; ++x)
            affine = find(dhs[y], dws[x]) == t00 + y * wy + x * wx && dhs[y] == dhmin + y && dws[x] == (mode == 2 ? dwmin + x : gdw);
        if (!affine || t00 < 0 || t00 > 127 || wy > 127 || wx > 127 || wy < 0 || wx < 0) {
          nc = 7;
          break;
        }
        h.cp_ny[nc] = ndh;
        h.cp_nx[nc] = ndw;
        h.cp_w0[nc] = t00;
        h.cp_wy[nc] = wy;
        h.cp_wx[nc] = wx;
      }
      h.cp_map[nc] = m;
      h.cp_dw[nc] = gdw;
      h.cp_dh[nc] = dhmin;
      h.cp_ntaps[nc] = nt;
      h.cp_boxw[nc] = h.map_boxw[m];
      h.cp_boxh[nc] = h.map_boxh[m];
      ++nc;
    }
  }
  bool ok = nc >= 1 && nc <= 6 && n_ord == n_taps;
  for (int c = 0; ok && c < nc; ++c) ok = h.cp_boxw[c] <= 256 && h.cp_boxh[c] <= 256;
  if (!ok) return false;
  h.n_copies = nc;
  h.fused = 1;
  for (int c = 0; c < nc; ++c)
    if ((h.cp_boxw[c] * h.cp_boxh[c]) % 8 != 0) h.fused = 0;
  // candidate K chunks: the classic choice first, then smaller ones (they may let the weights stay resident)
  int bks[3], n_bk = 0;
  if (win > 0) bks[n_bk++] = cin;  // row-window stems: one chunk per filter row, trailing zero weight columns are skipped
  else {
    for (int c : {64, 32, 16})
      if (cin % c == 0 && (c >= 32 || n_bk == 0)) bks[n_bk++] = c;  // 16-wide chunks (32-byte rows) only when nothing else divides cin
  }
  // A/B knobs (read at every plan creation so one process can sweep them): K chunk, weight residency, CTAs per SM of the halo plans
  const int bk_env = [] { const char* e = getenv("CVB_HALO_BK"); return e ? atoi(e) : 0; }();
  const int res_env = [] { const char* e = getenv("CVB_HALO_RES"); return e ? atoi(e) : 1; }();
  const int ctas_env = [] { const char* e = getenv("CVB_HALO_CTAS"); return e ? atoi(e) : 0; }();
  const long long tiles_h = (long long)ceil_div(P.Wo, HTW) * ceil_div(P.Ho, HTH) * d->out.B * ceil_div(cout, bn);
  HaloCfg best;
  bool have = false;
  for (int ctas = 2; ctas >= 1; --ctas) {
    if (ctas == 2 && !(bn <= 64 && two_ctas_on())) continue;
    if (ctas_env && ctas != ctas_env) continue;
    if (!ctas_env && halo_req <= 0 && ctas == 1) continue;  // auto mode: only the two-CTAs-per-SM plans have been measured faster
    const int budget = ctas == 2 ? kSmemBudget2 : kSmemBudget;
    for (int bi = 0; bi < n_bk; ++bi) {
      const int bkh = bks[bi];
      if (bk_env && bkh != bk_env && win == 0) continue;
      if (!lookup_kernel(bn, bkh, P.f32)) continue;
      const ConvGeom g = conv_geom(bn, bkh, P.f32, false, false);
      const int swz = bkh * 2;
      const int chunks = cin / bkh;
      uint32_t slot = 0;
      double a_bytes = 0.0;
      HaloCfg cand = h;
      for (int c = 0; c < nc; ++c) {
        const int rows = cand.cp_boxw[c] * cand.cp_boxh[c];
        cand.cp_bytes[c] = (uint32_t)(rows * swz);
        cand.cp_lo_off[c] = (uint32_t)(((rows + 7) / 8 * 8) * swz);
        const uint32_t need = (cand.cp_lo_off[c] + cand.cp_bytes[c] + 1023u) / 1024u * 1024u;
        slot = need > slot ? need : slot;
        a_bytes += 2.0 * rows * swz;
      }
      a_bytes *= chunks;
      const int b_stage = 2 * g.b_bytes;
      const long long w_tot = (long long)n_taps * chunks * b_stage;
      const int kskip = win > 0 ? ((win - d->kw) * P.d.in.C) / 16 : 0;
      const double mma = ((double)n_taps * chunks * (bkh / 16 - kskip)) * kstep_clk;
      for (int cfg = 0; cfg < 4; ++cfg) {
        const int ob = (cfg & 2) ? 1 : 2;
        const int rt = (cfg & 1) ? 0 : 1;
        if (rt && !(P.has_resid && !P.f32 && resid_tma_on())) continue;
        for (int res = 1; res >= 0; --res) {
          int sa, sb = 0;
          if (res) {
            if (!(pin && !d->no_resident && res_env) || w_tot > budget) continue;
            sa = stages_fitting(budget, smem_layout(g, 0, (int)slot, (int)w_tot, ob, rt, false));
          } else {
            sb = 4;
            sa = stages_fitting(budget, smem_layout(g, 0, (int)slot, sb * b_stage, ob, rt, false));
            if (sa < 2) {
              sb = 3;
              sa = stages_fitting(budget, smem_layout(g, 0, (int)slot, sb * b_stage, ob, rt, false));
            }
          }
          if (sa < 2) continue;
          if (sa > 6) sa = 6;
          const double fill = (a_bytes + (res ? 0.0 : (double)w_tot)) / kFillBpc;
          double cost = (mma > fill ? mma : fill) + 300.0;
          cost *= (ctas == 2 ? 0.93 : 1.0) * (ob == 2 ? 0.97 : 1.0) * ((rt || !P.has_resid) ? 1.0 : 1.02) * (sa >= 3 ? 1.0 : 1.05) *
                  (bkh == 64 ? 1.0 : (bkh == 32 ? 1.01 : 1.03));
          if (!have || cost < best.cost) {
            best = cand;
            best.bk = bkh;
            best.resident = res;
            best.sa = sa;
            best.sb = sb;
            best.out_bufs = ob;
            best.resid_tma = rt;
            best.ctas = ctas;
            best.slot = slot;
            best.kskip = kskip;
            best.cost = cost;
            have = true;
          }
        }
      }
    }
  }
  if (!have) return false;
  // classic estimate: one 128-row box per (tap, chunk); weights resident only below 64 KB
  int cTW, cTH, cNB;
  choose_box(d->out.B, P.Ho, P.Wo, kTileM, &cTW, &cTH, &cNB);
  const long long tiles_c = (long long)ceil_div(P.Wo, cTW) * ceil_div(P.Ho, cTH) * ceil_div(d->out.B, cNB) * ceil_div(cout, bn);
  const int chunks_c = cin / bk;
  const long long w_c = (long long)n_taps * chunks_c * 2 * bn * bk * 2;
  const bool res_c = pin && !d->no_resident && w_c <= 64 * 1024;
  const double fill_c = ((double)n_taps * chunks_c * kTileM * bk * 4 + (res_c ? 0.0 : (double)w_c)) / kFillBpc;
  const double mma_c = (double)n_taps * cin / 16 * kstep_clk;
  const double cost_c = (double)tiles_c * ((mma_c > fill_c ? mma_c : fill_c) + 300.0);
  const double cost_h = (double)tiles_h * best.cost;
  if (!(halo_req > 0 || cost_h < 0.95 * cost_c)) return false;
  *out = best;
  return true;
}

// the fp32 accumulator tile of the epilogue shares the 227 KB with the ring: halve the K chunk until two streamed stages fit
static int fit_bk(int cin, int bn, int bk, bool f32, bool pp, bool rt) {
  while (bk > 16 && cin % (bk / 2) == 0 && lookup_kernel(bn, bk / 2, f32, false, 0, pp)) {
    const ConvGeom g = conv_geom(bn, bk, f32, false, pp);
    if (smem_layout(g, 2, 2 * g.a_bytes + 2 * g.b_bytes, 0, 1, rt, false).total <= kSmemBudget) break;
    bk /= 2;
  }
  return bk;
}

// ring of a plan: depth, slot bytes, resident weight slab, output staging buffers
struct Ring {
  int stages, resident, out_bufs, slot, weights;
};

// ring depth / resident weights / staging buffers of a classic-loader plan (geometry g, K chunk bk) that fit `budget` bytes of dynamic
// shared memory (0 stages = no fit)
static Ring plan_ring(const ConvProblem& P, int bn, const ConvGeom& g, int bk, bool rt, int budget) {
  const int k_it = P.n_taps * (P.cin / bk);
  const int a_st = 2 * g.a_bytes, b_st = 2 * g.b_bytes;
  const bool can_res = can_pin(P.cout, bn) && !P.d.no_resident && (long long)k_it * b_st <= 64 * 1024;
  auto fit = [&](int resident, int out_bufs) {
    Ring r{0, resident, out_bufs, resident ? a_st : a_st + b_st, resident ? k_it * b_st : 0};
    r.stages = stages_fitting(budget, smem_layout(g, 0, r.slot, r.weights, out_bufs, rt, false));
    return r;
  };
  if (can_res) {
    // the CTA's n-tile never changes and its whole weight slab fits: keep it resident, stream only activations
    const Ring r = fit(1, 2);
    if (r.stages >= 3 || (r.stages >= 2 && k_it == 1)) return r;
  }
  const Ring r2 = fit(0, 2);
  if (r2.stages >= 3) return r2;
  if (can_res) {
    const Ring r = fit(1, 1);
    if (r.stages >= 3) return r;
  }
  return fit(0, 1);
}

// K chunk, schedule, CTAs per SM and shared-memory plan of the layer
struct SchedPlan {
  int bk;
  bool pp;
  int ctas;  // CTAs per SM
  bool resid_tma;
  Ring ring;
  SmemLayout sm;
};

static int plan_schedule(const ConvProblem& P, int bn, int bk, const HaloCfg* hc, SchedPlan* S) {
  const CvbConvDesc* d = &P.d;
  const bool use_halo = hc != nullptr;
  const bool rt_on = resid_tma_on(), two_on = two_ctas_on();
  const bool rt = use_halo ? hc->resid_tma != 0 : (P.has_resid && !P.f32 && rt_on);  // the residual tile arrives by TMA
  if (use_halo) bk = hc->bk;
  // ---- CTAs per SM of the cooperative plan.  Narrow tiles whose ring, staging and accumulator tiles fit in half the shared memory
  // run two CTAs per SM, so one CTA's epilogue overlaps the other's main loop.  On the H100 every CTA also holds the fp32
  // accumulator tile, so most block_n = 64 plans do not fit and run one CTA per SM.
  Ring two{};
  bool two_ctas = use_halo && hc->ctas == 2;
  if (!use_halo && !P.yolo) {
    bk = fit_bk(P.cin, bn, bk, P.f32, false, rt);
    if (bn <= 64 && two_on && lookup_kernel(bn, bk, P.f32)) {
      two = plan_ring(P, bn, conv_geom(bn, bk, P.f32, false, false), bk, rt, kSmemBudget2);
      two_ctas = two.stages >= 3 || (two.stages >= 2 && two.out_bufs == 2);
    }
  }
  // ---- schedule.  Cooperative: both warpgroups share each 128-pixel tile and run its epilogue together, so the tensor pipe idles
  // during every epilogue (unless a second CTA on the SM fills it).  Ping-pong: 64-pixel tiles alternate between the warpgroups and one
  // warpgroup's epilogue overlaps the other's MMAs.  It streams each weight tile from L2 once per 64 instead of 128 pixels, but its
  // half-height activation stages also buy a deeper ring (or 64-wide K chunks) in the same shared memory.  Eligible: every one-CTA-per-SM
  // plan on the classic loader with block_n = 128, or with block_n <= 64 on a layer of at most 128 output channels -- the narrow plans
  // auto picks (narrow layers and the 128 -> 128 split).  A wider layer forced to narrow tiles would read every 64-pixel activation tile
  // from L2 once per n-tile; it has its 128-wide ping-pong plan, so the forced narrow plan stays cooperative.
  // Measured per layer on the YOLOv5-s stack (DESIGN.md 6): faster on every 1x1
  // layer.  Multi-tap layers depend on the width and the residual.  At block_n = 128, ping-pong is faster on every 3x3 and stride-2
  // layer except those with a residual, where the residual's staging tile leaves the ping-pong ring too shallow.  At block_n <= 64 it is
  // the other way round.  Ping-pong re-streams the whole weight slab per 64 pixels, and the 3x3 layers without a residual measured
  // 11-19 % slower.  With a residual, the cooperative ring is only two stages deep, and ping-pong measured 28 % faster.
  CVB_REQUIRE(d->schedule >= CVB_SCHED_AUTO && d->schedule <= CVB_SCHED_PINGPONG, "conv: schedule %d unsupported", d->schedule);
  const bool narrow_wide = bn < 128 && P.cout > 128;  // a layer of more than 128 channels in narrow n-tiles
  const bool pp_ok = !P.yolo && !use_halo && bn <= 128 && !narrow_wide && !two_ctas;
  CVB_REQUIRE(d->schedule != CVB_SCHED_PINGPONG || pp_ok,
              "conv: the ping-pong schedule needs a one-CTA-per-SM plan on the classic loader with block_n = 128, or block_n <= 64 on a "
              "layer of at most 128 channels (this plan %s)",
              P.yolo ? "runs the fused decode" : (use_halo ? "uses the halo loader" : (bn > 128 ? "has block_n = 256"
              : (narrow_wide ? "has narrow n-tiles on a layer of more than 128 channels"
              : "runs two CTAs per SM, which already overlap one CTA's epilogue with the other's MMAs"))));
  const bool pp_auto = P.n_taps == 1 || (bn == 128 ? !P.has_resid : P.has_resid);
  const bool pp = pp_ok && (d->schedule == CVB_SCHED_PINGPONG || (d->schedule == CVB_SCHED_AUTO && pp_auto));
  // a ping-pong plan runs one CTA per SM: no reason for the half-size K chunks of the narrow cooperative plans
  if (pp) bk = fit_bk(P.cin, bn, full_bk(P.cin), P.f32, true, rt);
  CVB_REQUIRE(lookup_kernel(bn, bk, P.f32, P.yolo, 0, pp), "conv: no kernel for block_n=%d block_k=%d yolo=%d", bn, bk, (int)P.yolo);

  // ---- shared-memory plan: ring depth, resident weights, output staging
  const ConvGeom g = conv_geom(bn, bk, P.f32, P.yolo, pp);
  int ctas = 1;
  Ring ring;
  if (P.yolo) {
    ring = Ring{0, 0, 1, 2 * g.a_bytes + 2 * g.b_bytes, 0};
    ring.stages = stages_fitting(kSmemBudget, smem_layout(g, 0, ring.slot, 0, 1, false, true));
    if (ring.stages > 4) ring.stages = 4;
  } else if (use_halo) {
    const int w_stage = 2 * g.b_bytes;
    ring = Ring{hc->sa, hc->resident, hc->out_bufs, (int)hc->slot, hc->resident ? P.n_taps * (P.cin / bk) * w_stage : hc->sb * w_stage};
    ctas = hc->ctas;
  } else if (two_ctas) {
    // the cooperative narrow plan that fits half the SM's shared memory (decided with the schedule above)
    ring = two;
    ctas = 2;
  } else {
    ring = plan_ring(P, bn, g, bk, rt, kSmemBudget);
  }
  if (ring.stages > 8) ring.stages = 8;
  CVB_REQUIRE(ring.stages >= 2, "conv: tile does not fit in shared memory (block_n=%d block_k=%d)", bn, bk);
  S->bk = bk;
  S->pp = pp;
  S->ctas = ctas;
  S->resid_tma = rt;
  S->ring = ring;
  S->sm = smem_layout(g, ring.stages, ring.slot, ring.weights, ring.out_bufs, rt, P.yolo);
  // the layout must fit the budget it was sized for, start its ring slots on the swizzle atom, and leave room for every mbarrier (full /
  // empty per ring slot and per halo weight slot, resident weights, two residual tiles)
  const int budget = ctas == 2 ? kSmemBudget2 : kSmemBudget;
  CVB_REQUIRE(S->sm.total <= budget && S->sm.slot % 1024 == 0,
              "conv: internal error (shared-memory layout of %d bytes, ring slot %d, for a budget of %d)", S->sm.total, S->sm.slot, budget);
  const int bars = 2 * ring.stages + 2 * (use_halo ? hc->sb : 0) + 3;
  CVB_REQUIRE(bars <= kMaxBars, "conv: internal error (%d mbarriers, room for %d)", bars, kMaxBars);
  return CVB_OK;
}

// ---- tile box, tile counts and loader arguments
static void fill_tiles(const ConvProblem& P, const TapTable& T, int bn, const SchedPlan& S, const HaloCfg* hc, ConvKArgs& a) {
  const int bk = S.bk;
  const int tile_m = S.pp ? kTileM / 2 : kTileM;  // output pixels of one tile
  int TW, TH, NB;
  choose_box(P.d.out.B, P.Ho, P.Wo, tile_m, &TW, &TH, &NB);
  if (P.yolo) {  // one image per tile (the epilogue keeps a per-image histogram), 128 consecutive pixels of the flattened level
    TW = P.Wo < kTileM ? P.Wo : kTileM;
    TH = 1;
    NB = 1;
  }
  if (hc) {
    TW = kHaloTW;
    TH = kHaloTH;
    NB = 1;
  }
  a.TW = TW;
  a.TH = TH;
  a.NB = NB;
  a.tiles_w = ceil_div(P.Wo, TW);
  a.tiles_h = ceil_div(P.Ho, TH);
  a.tiles_b = ceil_div(P.d.out.B, NB);
  a.tiles_n = ceil_div(P.cout, bn);
  {
    const unsigned long long total_t = (unsigned long long)a.tiles_w * a.tiles_h * a.tiles_b * a.tiles_n;
    a.mg_n = fast_div_magic(a.tiles_n, total_t);
    a.mg_w = fast_div_magic(a.tiles_w, total_t);
    a.mg_h = fast_div_magic(a.tiles_h, total_t);
  }
  a.Ho = P.Ho;
  a.Wo = P.Wo;
  a.Bn = P.d.out.B;
  a.cout = P.cout;
  a.taps = P.n_taps;
  a.chunks = P.cin / bk;
  a.cin = P.cin;
  a.act = P.d.act;
  a.rows_valid = TW * TH * NB;
  a.a_box_bytes = (uint32_t)(TW * TH * NB * bk * 2);
  a.a_fused = (a.rows_valid % 8 == 0) ? 1 : 0;  // the lo plane must start on a swizzle-atom boundary (8 rows)
  a.a_lo_off = a.a_fused ? a.a_box_bytes : (uint32_t)(tile_m * bk * 2);
  a.bias = P.d.bias;
  a.bias_len = P.d.cout_pad;
  a.stages = S.ring.stages;
  a.b_resident = S.ring.resident;
  a.out_bufs = S.ring.out_bufs;
  a.sm = S.sm;
  for (int t = 0; t < P.n_taps; ++t) {
    a.tap_map[t] = T.map[t];
    a.tap_dh[t] = T.dh[t];
    a.tap_dw[t] = T.dw[t];
  }
  if (hc) {
    a.halo = hc->mode;
    a.n_copies = hc->n_copies;
    a.sb_stages = hc->sb;
    a.kskip = hc->kskip;
    a.a_fused = hc->fused;
    for (int c = 0; c < hc->n_copies; ++c) {
      a.cp_map[c] = (int8_t)hc->cp_map[c];
      a.cp_dw[c] = (int8_t)hc->cp_dw[c];
      a.cp_dh[c] = (int8_t)hc->cp_dh[c];
      a.cp_ntaps[c] = (int8_t)hc->cp_ntaps[c];
      a.cp_bytes[c] = hc->cp_bytes[c];
      a.cp_lo_off[c] = hc->fused ? hc->cp_bytes[c] : hc->cp_lo_off[c];
      a.cp_sbo[c] = (uint32_t)(hc->cp_boxw[c] * bk * 2);  // 8 consecutive accumulator rows = 8 horizontally adjacent pixels (TW == 8)
      a.cp_ny[c] = (int8_t)hc->cp_ny[c];
      a.cp_nx[c] = (int8_t)hc->cp_nx[c];
      a.cp_w0[c] = (int8_t)hc->cp_w0[c];
      a.cp_wy[c] = (int8_t)hc->cp_wy[c];
      a.cp_wx[c] = (int8_t)hc->cp_wx[c];
      a.cp_row16[c] = (uint32_t)(hc->cp_boxw[c] * bk * 2) >> 4;
    }
    for (int t = 0; t < P.n_taps; ++t) {
      a.tap_w[t] = (int8_t)hc->tap_w[t];
      a.tap_off[t] = (uint16_t)hc->tap_off[t];
    }
  }
}

// ---- tensor maps: input (5D: C, W, H, B, plane), weights (3D: K, cout_pad, plane), output and residual (5D)
static int encode_maps(const ConvProblem& P, int bn, const SchedPlan& S, const HaloCfg* hc, ConvKArgs& a) {
  const CvbConvDesc* d = &P.d;
  const CvbView& in = d->in;
  const CvbView& out = d->out;
  const int bk = S.bk, cin = P.cin, Wo = P.Wo, Ho = P.Ho;
  const CUtensorMapDataType f16 = CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  int box[5] = {bk, a.TW, a.TH, a.NB, a.a_fused ? 2 : 1};
  if (hc) {
    box[1] = hc->map_boxw[0];
    box[2] = hc->map_boxh[0];
  }
  const long long pix = (long long)in.c_pitch * 2;  // bytes per pixel
  int rc = CVB_OK;
  if (d->stride == 1) {
    // window mode (win > 0): overlapping-window view, element (k, w, h, b, p) = padded_input[p][b][h][w + k / C][k % C];
    // consecutive w overlap
    rc = encode_5d(&a.tmA[0], f16, in.base, cin, P.win > 0 ? Wo : in.W, in.H, in.B, 2, pix, pix * in.W, pix * in.W * in.H,
                   in.plane_stride, box, swizzle_for_bytes(bk * 2));
  } else {
    for (int py = 0; py < 2 && rc == CVB_OK; ++py)
      for (int px = 0; px < 2 && rc == CVB_OK; ++px) {
        const int Wp = (in.W - px + 1) / 2, Hp = (in.H - py + 1) / 2;  // number of columns/rows with this parity
        if (Wp <= 0 || Hp <= 0) {
          a.tmA[py * 2 + px] = a.tmA[0];
          continue;
        }
        if (hc && hc->map_boxw[py * 2 + px] > 0) {
          box[1] = hc->map_boxw[py * 2 + px];
          box[2] = hc->map_boxh[py * 2 + px];
        }
        const uint8_t* base = static_cast<const uint8_t*>(in.base) + ((long long)py * in.W + px) * pix;
        rc = encode_5d(&a.tmA[py * 2 + px], f16, base, cin, Wp, Hp, in.B, 2, pix * 2, pix * in.W * 2, pix * in.W * in.H, in.plane_stride,
                       box, swizzle_for_bytes(bk * 2));
      }
  }
  if (rc == CVB_OK) {
    const long long K = (long long)a.taps * cin;
    const cuuint64_t dims[3] = {(cuuint64_t)K, (cuuint64_t)d->cout_pad, 2};
    const cuuint64_t str[2] = {(cuuint64_t)(K * 2), (cuuint64_t)(K * 2 * d->cout_pad)};
    const cuuint32_t wbox[3] = {(cuuint32_t)bk, (cuuint32_t)bn, 2};
    rc = encode_map(&a.tmB, f16, 3, d->weights, dims, str, wbox, swizzle_for_bytes(bk * 2));
  }
  // output and residual tiles: one output group of the tile box (fp32: one plane)
  const ConvGeom g = conv_geom(bn, bk, P.f32, P.yolo, S.pp);
  const int obox[5] = {g.out_group_ch, a.TW, a.TH, a.NB, 1};
  if (rc == CVB_OK && !P.yolo) {
    const long long opix = (long long)out.c_pitch * (P.f32 ? 4 : 2);
    rc = encode_5d(&a.tmO, P.f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : f16, out.base, P.cout, Wo, Ho, out.B, P.f32 ? 1 : 2, opix, opix * Wo,
                   opix * Wo * Ho, P.f32 ? opix * Wo * Ho * out.B : out.plane_stride, obox, swizzle_for_bytes(g.out_row_bytes));
  }
  if (rc == CVB_OK && S.resid_tma) {  // the residual tile: same box / swizzle as the output tile
    const CvbView& r = d->residual;
    const long long rpix = (long long)r.c_pitch * 2;
    rc = encode_5d(&a.tmR, f16, r.base, P.cout, Wo, Ho, out.B, 2, rpix, rpix * Wo, rpix * Wo * Ho, r.plane_stride, obox,
                   swizzle_for_bytes(g.out_row_bytes));
  }
  return rc;
}

// ---- epilogue operands, fused-decode arguments, accumulation gain; returns the kernel (compile-time epilogue specialisation)
static const void* fill_epilogue(const ConvProblem& P, int bn, const SchedPlan& S, ConvKArgs& a, int* epi_out) {
  const CvbConvDesc* d = &P.d;
  if (d->residual.base) {
    const CvbView& r = d->residual;
    a.resid = static_cast<const __half*>(r.base);
    a.resid_plane = r.plane_stride / 2;
    a.resid_pitch = r.c_pitch;
    a.resid_tma = S.resid_tma ? 1 : 0;
    a.resid_first = d->residual_before_act ? 1 : 0;
    a.resid_scale = d->residual_scale != 0.0f ? d->residual_scale : 1.0f;
  }
  if (d->up_partial.base) {
    const CvbView& u = d->up_partial;
    a.up = static_cast<const float*>(u.base);
    a.up_pitch = u.c_pitch;
    a.up_H = u.H;
    a.up_W = u.W;
  }
  if (P.yolo) {
    const CvbYoloDecode& y = *d->yolo;
    a.tile_contig = 1;
    a.yz = y.z;
    a.y_zrows = y.z_rows;
    a.y_zoff = y.z_off;
    a.y_no = y.no;
    a.y_nx = P.yolo_nx;
    a.y_nx_magic = (uint32_t)((0x100000000ULL + (unsigned long long)P.yolo_nx - 1) / (unsigned long long)P.yolo_nx);
    a.y_multi = y.multi_label && y.no - 5 > 1 ? 1 : 0;
    a.y_stride = y.stride;
    a.y_conf = y.conf_thres;
    for (int i = 0; i < 8; ++i) a.y_anchor[i] = y.anchors_px[i];
    a.y_hist = static_cast<unsigned int*>(y.nms_workspace);
    a.y_rowmax = nms_ws_rowmax(y.nms_workspace, d->out.B);
  }
  {
    // one accumulation chain per tile: the hi*hi products (and, at block_n = 256, the cross terms too: one register accumulator) of
    // every K step; rz_gain undoes the mean round-toward-zero shrink of the chain
    const int chain = (bn <= 128 ? 1 : 3) * a.taps * P.cin / 16;
    static const double rz_c = [] {
      // mean |sum| shrink per chained MMA of the tensor core's round-toward-zero fp32 accumulation (tools/precision_probe.py);
      // CVB_RZ_COMP overrides it
      const char* e = getenv("CVB_RZ_COMP");
      return e ? atof(e) : 1.9e-8;
    }();
    a.rz_gain = (float)(1.0 + rz_c * (double)chain);
  }
  // compile-time specialised epilogues for the two hot modes (same tile / smem geometry as the generic kernel)
  static const bool spec_on = [] { const char* e = getenv("CVB_EPI_SPEC"); return !(e && atoi(e) == 0); }();  // A/B knob
  int epi = 0;
  if (spec_on && !P.f32 && !P.yolo && !d->up_partial.base) {
    if (d->act == CVB_ACT_SILU) {
      if (!d->residual.base) epi = 1;
      else if (a.resid_tma && !a.resid_first && a.resid_scale == 1.0f) epi = 2;
    } else if (d->act == CVB_ACT_RELU) {
      if (!d->residual.base) epi = 3;
      else if (a.resid_tma && a.resid_first && a.resid_scale == 1.0f) epi = 4;
    }
  }
  const void* fn = epi ? lookup_kernel(bn, S.bk, P.f32, false, epi, S.pp, S.ctas) : nullptr;
  *epi_out = fn ? epi : 0;
  return fn ? fn : lookup_kernel(bn, S.bk, P.f32, P.yolo, 0, S.pp, S.ctas);
}

// programmatic dependent launch (prologue of conv N+1 overlapping the tail of conv N): measured neutral on the YOLOv5-s step (6.57 vs
// 6.55 ms; the persistent grids leave no idle SMs to overlap into), so it stays opt-in: CVB_PDL=1
static bool pdl_on() {
  static const bool on = [] {
    const char* e = getenv("CVB_PDL");
    return e && atoi(e) == 1;
  }();
  return on;
}

// ---- diagnostics switches and the persistent launch grid
static int set_launch(const ConvProblem& P, int bn, const SchedPlan& S, CvbConvPlan* p) {
  ConvKArgs& a = p->args;
  {
    const char* e = getenv("CVB_DBG");  // diagnostics only (tools/conv_pipeline_profile.py): results are wrong when set
    a.dbg = e ? atoi(e) : 0;
    static const int hint = [] {
      const char* h = getenv("CVB_WAIT_HINT");  // tuning knob: ns the producer may sleep per free-slot wait (default 0 = spin)
      return h ? atoi(h) : 0;
    }();
    a.wait_hint = (uint32_t)(hint > 0 ? hint : 0);
  }
  p->smem = S.sm.total;
  p->threads = kThreads;
  p->schedule = S.pp ? CVB_SCHED_PINGPONG : CVB_SCHED_COOPERATIVE;
  int sms = sm_count();
  if (sms == 0) return CVB_ERR_NO_DEVICE;
  CVB_CHECK_CUDA(opt_in_smem(p->fn, kSmemBudget));
  const long long total = (long long)a.tiles_w * a.tiles_h * a.tiles_b * a.tiles_n;
  if (P.d.sm_limit > 0 && P.d.sm_limit < sms) sms = P.d.sm_limit;
  sms *= S.ctas;
  p->grid = (int)(total < sms ? total : sms);
  if (a.b_resident && a.tiles_n > 1) {
    p->grid -= p->grid % a.tiles_n;  // every CTA keeps one n-tile (tile % tiles_n constant along its stride)
    if (p->grid < a.tiles_n) p->grid = a.tiles_n;
  }
  static const bool dbg = [] { const char* e = getenv("CVB_PLAN_DEBUG"); return e && atoi(e) != 0; }();
  if (dbg)
    fprintf(stderr, "[cvb plan] cin=%d cout=%d k=%dx%d s=%d out=%dx%dx%d bn=%d bk=%d stages=%d resident=%d out_bufs=%d ctas/sm=%d "
            "smem=%d grid=%d tiles=%lld resid_tma=%d halo=%d copies=%d sb=%d slot=%u kskip=%d schedule=%s epi=%d f32=%d yolo=%d pdl=%d\n", P.cin, P.cout,
            P.d.kh, P.d.kw, P.d.stride, P.d.out.B, P.Ho, P.Wo, bn, S.bk, a.stages, a.b_resident, a.out_bufs, S.ctas, p->smem, p->grid, total,
            a.resid_tma, a.halo, a.n_copies, a.sb_stages, a.halo ? (unsigned)a.sm.slot : 0u, a.kskip, S.pp ? "pingpong" : "cooperative",
            p->epi, (int)P.f32, (int)P.yolo, (int)pdl_on());
  return CVB_OK;
}

}  // namespace cvb

extern "C" int cvb_conv_plan_create(const CvbConvDesc* desc, CvbConvPlan** out_plan) {
  using namespace cvb;
  CVB_REQUIRE(desc != nullptr && out_plan != nullptr, "null argument");
  *out_plan = nullptr;
  ConvProblem P;
  int rc = validate_desc(*desc, &P);
  if (rc != CVB_OK) return rc;
  int bn, bk;
  if ((rc = choose_block(P, &bn, &bk)) != CVB_OK) return rc;
  TapTable taps;
  if ((rc = build_taps(P, &taps)) != CVB_OK) return rc;
  HaloCfg hc;
  const HaloCfg* halo = plan_halo(P, taps, bn, bk, &hc) ? &hc : nullptr;
  SchedPlan S;
  if ((rc = plan_schedule(P, bn, bk, halo, &S)) != CVB_OK) return rc;
  std::unique_ptr<CvbConvPlan> p(new (std::nothrow) CvbConvPlan());
  CVB_REQUIRE(p != nullptr, "out of host memory");
  memset(&p->args, 0, sizeof(p->args));
  fill_tiles(P, taps, bn, S, halo, p->args);
  rc = encode_maps(P, bn, S, halo, p->args);
  if (rc != CVB_OK) return rc;
  p->fn = fill_epilogue(P, bn, S, p->args, &p->epi);
  rc = set_launch(P, bn, S, p.get());
  if (rc != CVB_OK) return rc;
  *out_plan = p.release();
  return CVB_OK;
}

extern "C" int cvb_conv_plan_run(const CvbConvPlan* p, void* stream) {
  using namespace cvb;
  CVB_REQUIRE(p != nullptr, "null plan");
  void* kargs[1] = {const_cast<ConvKArgs*>(&p->args)};
  const bool pdl = pdl_on();
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(p->grid);
  cfg.blockDim = dim3(p->threads);
  cfg.dynamicSmemBytes = (size_t)p->smem;
  cfg.stream = as_stream(stream);
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  CVB_CHECK_CUDA(cudaLaunchKernelExC(&cfg, p->fn, kargs));
  count_launch();
  return CVB_OK;
}

extern "C" int cvb_conv_plan_run_many(CvbConvPlan* const* plans, int32_t n, void* stream) {
  for (int i = 0; i < n; ++i) {
    int rc = cvb_conv_plan_run(plans[i], stream);
    if (rc != CVB_OK) return rc;
  }
  return CVB_OK;
}

extern "C" void cvb_conv_plan_destroy(CvbConvPlan* p) { delete p; }

extern "C" int cvb_conv_plan_set_profile(CvbConvPlan* p, long long* counters, int32_t* grid) {
  CVB_REQUIRE(p != nullptr, "null plan");
  p->args.prof = counters;
  if (grid) *grid = p->schedule == CVB_SCHED_PINGPONG ? 2 * p->grid : p->grid;  // counter rows: one per warpgroup in ping-pong
  return CVB_OK;
}
