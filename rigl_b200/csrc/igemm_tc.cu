// Masked conv2d / linear as implicit GEMM on the Hopper tensor cores (sm_90a, wgmma).
//
//   fprop : y[pix, co]  = sum_{tap, ci} x[pix (+) tap, ci] * Wm[tap][co][ci]
//   dgrad : dx[pix, ci] = sum_{tap, co} dy[pix (-) tap, co] * Wm[tap][ci][co]
//   wgrad : dW[tap][ci][co] = sum_{pix} x[pix (+) tap, ci] * dy[pix, co]      (dense, fp32)
// Wm = mask * W is produced once per step by pack.cu; its per-tile survivor counts
// gate the weight-tile loads (an all-zero 64x64 weight tile costs no TMA and no MMA).
//
// No im2col buffer (except the 3-channel stem's patch matrix, conv_simt.cu): an M tile is a BOX of 128 output pixels
// (bw x bh x bn over width, height, batch) and, for filter tap (kh,kw), the A
// operand is the same box shifted by the tap offset, fetched by ONE 4-D TMA
// (cp.async.bulk.tensor.4d) whose out-of-bounds zero fill implements the padding.
// Stride-2 convs read through four parity sub-grid tensor maps (same trick,
// element strides doubled), so every conv shape in ResNet/WRN is a plain loop of
// TMA boxes + wgmma.mma_async with fp32 accumulators in registers.
//
// Kernel organisation (persistent, one CTA per SM, 384 threads = three warpgroups):
//   warp 0        : TMA producer (converged warp, one elected lane issues)   smem ring, full/empty mbarriers
//   warpgroups 1-2: consumers: each issues the wgmma for 64 of the tile's 128 rows, then runs the epilogue of
//                   those rows from its registers: bf16 -> swizzled smem slab -> TMA store (or direct fp32/bias
//                   stores); the producer refills the ring for the next tile meanwhile.
// Variants: k_igemm_kmajor (fprop/dgrad, optional fused BN statistics), k_igemm_wgrad, and -- textually included
// below -- halo3x3.cuh (3x3/s1 layers with <= 64 channels: one smem halo tile feeds all nine taps) and
// stem_s2d.cuh (the 7x7/2 stem).  DESIGN.md 3 describes the design.
// fprop/dgrad use K-major operands; wgrad reduces over pixels, so both operands are
// MN-major views of the NHWC tensors (no transposes are materialised) and the
// pixel range is split across CTAs (deterministic two-pass split-K).
#include <cuda.h>
#include <cuda_bf16.h>

#include <stdio.h>
#include <stdlib.h>

#include <mutex>

#include "common.cuh"
#include "conv_common.cuh"
#include "tc_ptx.cuh"

namespace rigl {

using namespace ptx;

constexpr int kMaxTaps = 9;
constexpr int kBM = 128;            // M tile: two warpgroups x 64 rows
constexpr int kBK = 64;             // K block: 64 bf16 = one 128B swizzle row
constexpr int kThreads = 384;       // warpgroup 0: producer; warpgroups 1-2: consumers
constexpr int kConsumerWarp0 = 4;
constexpr int kConsumerWarps = 8;
constexpr int kConsumerThreads = 256;

struct TapInfo {
  int8_t map_id, dh, dw, pad;
  int32_t b_tap;                    // tap index into the packed weights
};

struct IgemmParams {
  int ntaps;
  TapInfo taps[kMaxTaps];
  int kblks;                        // K blocks per tap
  int GW, GH, NB;                   // pixel grid covered by this launch
  int bw, bh, bn;                   // pixel box of one M tile (bw*bh*bn == 128)
  int tiles_w, tiles_h, tiles_n;    // boxes per dimension
  int n_tiles;                      // tiles along the output-channel dim
  int N;                            // output channels
  __nv_bfloat16* out_bf16;
  float* out_f32;
  const float* bias;
  long long o_off, o_sn, o_sh, o_sw;   // element offsets of pixel (n,h,w) in the output
  const uint32_t* nnz;              // survivor counts per 64x64 weight tile (or null)
  int nnz_tap_stride, nnz_n_stride, nnz_k_stride;
  int tma_store;                    // 1: epilogue stages bf16 tiles in smem and TMA-stores them
  float* bn_partial;                // optional [gridDim.x][2][N]: per-CTA column sums / sums of squares of D
};

// Inference batch norm applied by the epilogue of k_igemm_kmajor_bn (TMA-store path only).
struct BnEpilogue {
  const float* scale;               // [N]
  const float* shift;               // [N]
  int relu;
  int residual;                     // 1: the residual box is TMA-loaded into the staging slab before it is staged
};

struct TMaps4 {
  CUtensorMap a[4];
};

__device__ __forceinline__ bool weight_block_live(const IgemmParams& p, int tap_idx, int n_tile, int kb, int bn64) {
  if (p.nnz == nullptr) return true;
  const uint32_t* base = p.nnz + (long long)p.taps[tap_idx].b_tap * p.nnz_tap_stride + (long long)kb * p.nnz_k_stride;
  uint32_t s = 0;
  for (int j = 0; j < bn64; ++j) {
    const int nt = n_tile * bn64 + j;
    if ((long long)nt * 64 < p.N) s += __ldg(base + (long long)nt * p.nnz_n_stride);
  }
  return s != 0;
}


// Liveness of every (tap, K block) of one N tile as a bitmask in shared memory, computed by a
// whole warp at the start of a tile (one round of parallel loads) instead of once per K block
// inside the issue loops, which are instruction-latency bound.  Block 0 is always live.
constexpr int kLiveWords = 10;        // 320 (tap, K block) pairs; longer reductions run without skipping
__device__ __forceinline__ bool live_mask_used(const IgemmParams& p) {   // no table (or too long): everything is live
  return p.nnz != nullptr && p.ntaps * p.kblks <= kLiveWords * 32;
}
template <int kBN64>
__device__ __forceinline__ bool build_live_mask(const IgemmParams& p, int n_tile, int lane, uint32_t* mask_smem) {
  const int nkb = p.ntaps * p.kblks;
  if (!live_mask_used(p)) return false;
  for (int w = 0; w * 32 < nkb; ++w) {
    const int j = w * 32 + lane;
    bool live = true;
    if (j > 0 && j < nkb) live = weight_block_live(p, j / p.kblks, n_tile, j % p.kblks, kBN64);
    const uint32_t m = __ballot_sync(0xffffffffu, live);
    if (lane == 0) mask_smem[w] = m;
  }
  __syncwarp();
  return true;
}

// ----------------------------------------------------------------------------
// fprop / dgrad kernel: D[128 pixels, BN] += A[128, 64] * B[BN, 64]^T per (tap, k block)
// ----------------------------------------------------------------------------
// Batch-norm statistics of one staged output slab (128 pixel rows x 64 channels, bf16, 128-byte rows with the
// 16-byte chunks XOR-swizzled by row & 7 -- exactly what the TMA store is about to read): column sums and sums of
// squares of the values AS STORED (bf16-rounded), added to this CTA's row of the partial table.
//   warp q (0..3) owns channels 16q..16q+15 (chunks 2q, 2q+1); lane = (row group g = lane >> 3, channel pair
//   cp = lane & 7); group g walks rows 32g + ((i + 2g) & 31), i = 0..31: the four groups then sit on four different
//   swizzle phases, so the 32 lanes of every LDS.32 hit 32 different banks.
// 32 LDS + ~130 FP ops per thread per slab, two shuffles per statistic, and ONE RED per (slab, channel, statistic):
// each table entry is only ever touched by one lane of one warp, in tile order, so the fp32 sums are deterministic.
// Rows outside the pixel grid are written as zeros by their owner (see stage_slab), so they do not count.
__device__ __forceinline__ void slab_bn_stats(uint32_t slab, int quad, int lane, float* __restrict__ bn_row, int co0,
                                              int n) {
  const int cp = lane & 7, g = lane >> 3;
  const uint32_t chunk = (uint32_t)(2 * quad + (cp >> 2));
  const uint32_t word = (uint32_t)(cp & 3) * 4u;
  float s0 = 0.f, s1 = 0.f, q0 = 0.f, q1 = 0.f;
#pragma unroll 8
  for (int i = 0; i < 32; ++i) {
    const uint32_t row = (uint32_t)(32 * g + ((i + 2 * g) & 31));
    uint32_t v;
    asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(slab + row * 128u + (((chunk ^ (row & 7u)) << 4) | word)));
    const float a = __uint_as_float(v << 16), b = __uint_as_float(v & 0xffff0000u);
    s0 += a; s1 += b;
    q0 = fmaf(a, a, q0); q1 = fmaf(b, b, q1);
  }
#pragma unroll
  for (int o = 8; o <= 16; o <<= 1) {
    s0 += __shfl_xor_sync(0xffffffffu, s0, o); s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    q0 += __shfl_xor_sync(0xffffffffu, q0, o); q1 += __shfl_xor_sync(0xffffffffu, q1, o);
  }
  const int co = co0 + 16 * quad + 2 * cp;
  if (g == 0 && co < n) {          // (n is a multiple of 8 on this path, so co + 1 < n as well)
    atomicAdd(bn_row + co, s0); atomicAdd(bn_row + co + 1, s1);
    atomicAdd(bn_row + n + co, q0); atomicAdd(bn_row + n + co + 1, q1);
  }
}

// Accumulator fragment of a warpgroup's m64nN wgmma: register 4*j + 2*h + e holds
//   row 16 * (warp % 4) + lane / 4 + 8 * h,  column 8 * j + 2 * (lane % 4) + e.
// stage_slab writes columns [64 * S, 64 * S + 64) of this thread's two rows (tile rows `row` and `row + 8`) as bf16
// into a 128-row staging slab (128-byte rows, 16-byte chunks XOR-swizzled by row & 7, the TMA store's layout).
// Rows outside the output grid are written as zeros (they are clipped by the store but read by the statistics).
template <int S, int R>
__device__ __forceinline__ void stage_slab(const float (&d)[R], uint32_t slab, int row, bool ok0, bool ok1, int lane) {
#pragma unroll
  for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = row + 8 * h;
      const int e = 4 * (8 * S + jj) + 2 * h;
      __nv_bfloat162 v = __floats2bfloat162_rn(d[e], d[e + 1]);
      const uint32_t w = (h ? ok1 : ok0) ? *reinterpret_cast<uint32_t*>(&v) : 0u;
      const uint32_t dst = slab + (uint32_t)r * 128u + (uint32_t)((jj ^ (r & 7)) << 4) + (uint32_t)(lane & 3) * 4u;
      asm volatile("st.shared.b32 [%0], %1;" ::"r"(dst), "r"(w) : "memory");
    }
  }
}

// stage_slab with the inference batch norm applied: each stored pair is
//   [relu](fmaf(float(bf16_rn(D)), scale[c], shift[c]) [+ residual]) rounded to bf16,
// the arithmetic of bn.cu's bn_apply8 on exactly the value stage_slab would store, so the result is bit-identical
// to the plain fprop followed by rigl_bn_apply.  With `has_res` the slab already holds the residual box (TMA-loaded
// in the store's layout): every thread reads the words it is about to overwrite, and no other thread touches them.
// Coefficients of channels >= n (a ragged last slab) are not read; those columns are clipped by the store.
template <int S, int R>
__device__ __forceinline__ void stage_slab_bn(const float (&d)[R], uint32_t slab, int row, bool ok0, bool ok1, int lane,
                                              const BnEpilogue& ep, int co0, int n) {
#pragma unroll
  for (int jj = 0; jj < 8; ++jj) {
    const int co = co0 + 8 * jj + 2 * (lane & 3);
    float sc0 = 0.f, sc1 = 0.f, sh0 = 0.f, sh1 = 0.f;
    if (co < n) {                  // (n is a multiple of 8, so co + 1 < n as well)
      sc0 = __ldg(ep.scale + co); sc1 = __ldg(ep.scale + co + 1);
      sh0 = __ldg(ep.shift + co); sh1 = __ldg(ep.shift + co + 1);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = row + 8 * h;
      const int e = 4 * (8 * S + jj) + 2 * h;
      const uint32_t dst = slab + (uint32_t)r * 128u + (uint32_t)((jj ^ (r & 7)) << 4) + (uint32_t)(lane & 3) * 4u;
      const float2 f = __bfloat1622float2(__floats2bfloat162_rn(d[e], d[e + 1]));
      float a = fmaf(f.x, sc0, sh0), b = fmaf(f.y, sc1, sh1);
      if (ep.residual) {
        uint32_t rw;
        asm volatile("ld.shared.b32 %0, [%1];" : "=r"(rw) : "r"(dst) : "memory");
        a += __uint_as_float(rw << 16);
        b += __uint_as_float(rw & 0xffff0000u);
      }
      if (ep.relu) { a = fmaxf(a, 0.f); b = fmaxf(b, 0.f); }
      __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
      const uint32_t w = (h ? ok1 : ok0) ? *reinterpret_cast<uint32_t*>(&v) : 0u;
      asm volatile("st.shared.b32 [%0], %1;" ::"r"(dst), "r"(w) : "memory");
    }
  }
}

// stage_slab with a ReLU (VGG, whose convs have no batch norm):
//   fprop (kGate false): bf16(max(D, 0)), equal to relu of what stage_slab stores (rounding keeps the sign);
//   dgrad (kGate true):  the slab already holds the layer's forward input x (TMA-loaded in the store's layout, as the
//                        residual of stage_slab_bn); each stored value is bf16(D) where x > 0 and 0 elsewhere, the
//                        derivative of the ReLU that produced x.  Every thread reads the words it is about to overwrite.
template <int S, bool kGate, int R>
__device__ __forceinline__ void stage_slab_relu(const float (&d)[R], uint32_t slab, int row, bool ok0, bool ok1,
                                                int lane) {
#pragma unroll
  for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = row + 8 * h;
      const int e = 4 * (8 * S + jj) + 2 * h;
      const uint32_t dst = slab + (uint32_t)r * 128u + (uint32_t)((jj ^ (r & 7)) << 4) + (uint32_t)(lane & 3) * 4u;
      float a = d[e], b = d[e + 1];
      if (kGate) {
        uint32_t xw;
        asm volatile("ld.shared.b32 %0, [%1];" : "=r"(xw) : "r"(dst) : "memory");
        if (!(__uint_as_float(xw << 16) > 0.f)) a = 0.f;
        if (!(__uint_as_float(xw & 0xffff0000u) > 0.f)) b = 0.f;
      } else {
        a = fmaxf(a, 0.f); b = fmaxf(b, 0.f);
      }
      __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
      const uint32_t w = (h ? ok1 : ok0) ? *reinterpret_cast<uint32_t*>(&v) : 0u;
      asm volatile("st.shared.b32 [%0], %1;" ::"r"(dst), "r"(w) : "memory");
    }
  }
}

template <int R>
__device__ __forceinline__ void zero_acc(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) d[i] = 0.f;
}

// Warp roles (384 threads, one CTA per SM, persistent over tiles):
//   warp 0       : TMA producer (converged warp, one elected lane issues)   smem ring, full/empty mbarriers
//   warps 1-3    : idle
//   warps 4-11   : two consumer warpgroups; warpgroup w issues the wgmma of pixel rows 64w..64w+63 of the tile
//                  (A from shared memory, K-major), keeps its 64 x BN fp32 accumulators in registers, then runs
//                  the epilogue for those rows: bf16 -> swizzled smem slab -> TMA store (or direct fp32/bias
//                  stores).  The producer keeps filling the ring for the next tile meanwhile.
// A stage is refilled once every consumer warp has arrived on its empty barrier.
// kEpi selects the epilogue at compile time:
//   kEpiPlain     stage_slab (or direct stores), optional BN statistics;
//   kEpiBn        the inference batch norm (stage_slab_bn); with ep.residual the residual box at the output tile's
//                 coordinates is first TMA-loaded into the staging slab (one more mbarrier, no more shared memory);
//   kEpiRelu      fprop with the ReLU applied (stage_slab_relu);
//   kEpiReluGate  dgrad gated by the layer's forward input, TMA-loaded through *rmap like the residual.
constexpr int kEpiPlain = 0, kEpiBn = 1, kEpiRelu = 2, kEpiReluGate = 3;
template <int BN, int STAGES, int kEpi>
__device__ __forceinline__ void kmajor_body(const TMaps4& amaps, const CUtensorMap& bmap, const CUtensorMap& omap,
                                            const IgemmParams& p, const CUtensorMap* rmap, const BnEpilogue& ep) {
  constexpr bool kBnApply = kEpi == kEpiBn;
  constexpr bool kLoadsSlab = kEpi == kEpiBn || kEpi == kEpiReluGate;   // the residual / gate box barrier exists
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  constexpr uint32_t kABytes = kBM * kBK * 2;        // 16 KB
  constexpr uint32_t kBBytes = BN * kBK * 2;
  constexpr uint32_t kStageBytes = kABytes + kBBytes;
  constexpr uint32_t kSlabBytes = kBM * 64 * 2;       // one 128-pixel x 64-channel output slab
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t out_base = smem_base + STAGES * kStageBytes;          // 2 staging slabs (1024B aligned)
  const uint32_t bar_base = out_base + 2 * kSlabBytes;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };
  const uint32_t res_bar = bar_base + 8u * (2 * STAGES);             // kLoadsSlab: residual / gate box loaded

  // live_cons[warpgroup][tile parity]: one liveness mask per consumer warpgroup, double-buffered over tiles
  __shared__ uint32_t live_prod[kLiveWords], live_cons[2][2][kLiveWords];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < 4; ++i) prefetch_tmap(&amaps.a[i]);
    prefetch_tmap(&bmap);
    if (p.tma_store) prefetch_tmap(&omap);
    for (int s = 0; s < STAGES; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), kConsumerWarps); }
    if constexpr (kLoadsSlab) {
      mbar_init(res_bar, 1);
      if (kEpi == kEpiReluGate || ep.residual) prefetch_tmap(rmap);
    }
    fence_barrier_init();
  }
  __syncthreads();

  // Tile schedule: tiles are dealt round-robin to CTAs, N fastest (neighbouring CTAs reuse the same activation tiles
  // in L2).
  const int m_tiles = p.tiles_w * p.tiles_h * p.tiles_n;
  const int total = m_tiles * p.n_tiles;
  const int first = blockIdx.x, step = gridDim.x;
  constexpr int kBN64 = (BN + 63) / 64;

  if (warp == 0) {
    // ===================== TMA producer (converged warp, one elected lane issues) =====================
    int stage = 0; uint32_t phase = 0;
    for (int tile = first; tile < total; tile += step) {
      const int n_tile = tile % p.n_tiles;
      const int m_tile = tile / p.n_tiles;
      const int tw = m_tile % p.tiles_w;
      const int th = (m_tile / p.tiles_w) % p.tiles_h;
      const int tn = m_tile / (p.tiles_w * p.tiles_h);
      const bool masked = build_live_mask<kBN64>(p, n_tile, lane, live_prod);
      int j = 0;
      for (int t = 0; t < p.ntaps; ++t) {
        const TapInfo tap = p.taps[t];
        for (int kb = 0; kb < p.kblks; ++kb, ++j) {
          if (masked && !((live_prod[j >> 5] >> (j & 31)) & 1u)) continue;
          mbar_wait(empty_bar(stage), phase ^ 1u);
          if (elect_one()) {
            const uint32_t a_dst = smem_base + stage * kStageBytes;
            mbar_arrive_expect_tx(full_bar(stage), kStageBytes);      // A + B
            tma_load_4d(a_dst, &amaps.a[tap.map_id], full_bar(stage), kb * kBK, tw * p.bw + tap.dw,
                        th * p.bh + tap.dh, tn * p.bn);
            tma_load_3d(a_dst + kABytes, &bmap, full_bar(stage), kb * kBK, n_tile * BN, tap.b_tap);
          }
          __syncwarp();
          if (++stage == STAGES) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else if (warp >= kConsumerWarp0) {
    // ===================== consumers: wgmma main loop + epilogue =====================
    const int cw = warp - kConsumerWarp0;                 // 0..7
    const int wg = cw >> 2;                               // 64-row half of the tile
    const int row = 64 * wg + 16 * (cw & 3) + (lane >> 2);   // this thread's first tile row (second: row + 8)
    const bool issuer = (cw == 0 && lane == 0);
    float acc[BN / 2];
    int stage = 0; uint32_t phase = 0;
    uint32_t slab_ctr = 0;
    uint32_t res_phase = 0;
    float* bn_row = (kEpi == kEpiPlain && p.bn_partial) ? p.bn_partial + (size_t)blockIdx.x * 2 * p.N : nullptr;
    if (bn_row) {            // this CTA's row of the batch-norm partial sums starts at zero
      for (int i = cw * 32 + lane; i < 2 * p.N; i += kConsumerThreads) bn_row[i] = 0.f;
      __threadfence_block();
      named_bar_sync(1, kConsumerThreads);
    }
    int tile_ctr = 0;
    for (int tile = first; tile < total; tile += step, ++tile_ctr) {
      const int n_tile = tile % p.n_tiles;
      const int m_tile = tile / p.n_tiles;
      // the first warp of the warpgroup builds the tile's liveness mask, the other three wait for it
      uint32_t* live = live_cons[wg][tile_ctr & 1];
      if ((cw & 3) == 0) build_live_mask<kBN64>(p, n_tile, lane, live);
      named_bar_sync(3 + wg, 128);
      const bool masked = live_mask_used(p);
      zero_acc(acc);
      int prev = -1;
      const int nkb = p.ntaps * p.kblks;
      for (int j = 0; j < nkb; ++j) {
        if (masked && !((live[j >> 5] >> (j & 31)) & 1u)) continue;
        mbar_wait(full_bar(stage), phase);
        const uint32_t a_src = smem_base + stage * kStageBytes;
        const uint64_t da = make_smem_desc(a_src + (uint32_t)wg * 64u * 128u, 16, 1024);
        const uint64_t db = make_smem_desc(a_src + kABytes, 16, 1024);
        fence_regs(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBK / 16; ++k)              // +32 bytes along K = +2 in the 16-byte address field
          Wgmma<BN>::template ss<0, 0>(acc, da + 2 * k, db + 2 * k);
        wgmma_commit();
        wgmma_wait<1>();                                  // the previous stage's MMAs have read their operands
        if (prev >= 0 && lane == 0) mbar_arrive(empty_bar(prev));
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1u; }
      }
      wgmma_wait<0>();
      fence_regs(acc);
      if (prev >= 0 && lane == 0) mbar_arrive(empty_bar(prev));

      const int tw = m_tile % p.tiles_w;
      const int th = (m_tile / p.tiles_w) % p.tiles_h;
      const int tn = m_tile / (p.tiles_w * p.tiles_h);
      bool ok[2]; long long o_pix[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = row + 8 * h;
        const int pw = tw * p.bw + r % p.bw;
        const int ph = th * p.bh + (r / p.bw) % p.bh;
        const int pn = tn * p.bn + r / (p.bw * p.bh);
        ok[h] = pw < p.GW && ph < p.GH && pn < p.NB;
        o_pix[h] = p.o_off + pn * p.o_sn + ph * p.o_sh + pw * p.o_sw;
      }
      if (kEpi != kEpiPlain || p.tma_store) {
        // ---- stage 64-channel slabs in smem (128B-swizzled rows) and TMA-store them ----
#pragma unroll
        for (int s = 0; s < kBN64; ++s) {
          const int co0 = n_tile * BN + 64 * s;
          if (co0 >= p.N) break;                                   // uniform: whole slab out of range
          const uint32_t slab = out_base + (uint32_t)(slab_ctr & 1) * kSlabBytes;
          if (issuer) tma_store_wait_read<1>();                    // the store that last used this slab is done reading
          named_bar_sync(1, kConsumerThreads);
          if constexpr (kLoadsSlab) {
            if (kEpi == kEpiReluGate || ep.residual) {   // same box and swizzle as the store; rows outside the grid arrive as zeros
              if (issuer) {
                mbar_arrive_expect_tx(res_bar, kSlabBytes);
                tma_load_4d(slab, rmap, res_bar, co0, tw * p.bw, th * p.bh, tn * p.bn);
              }
              mbar_wait(res_bar, res_phase);
              res_phase ^= 1u;
            }
          }
          if constexpr (kBnApply) {
            if (s == 0) stage_slab_bn<0>(acc, slab, row, ok[0], ok[1], lane, ep, co0, p.N);
            else stage_slab_bn<(kBN64 > 1 ? 1 : 0)>(acc, slab, row, ok[0], ok[1], lane, ep, co0, p.N);
          } else if constexpr (kEpi != kEpiPlain) {
            constexpr bool kGate = kEpi == kEpiReluGate;
            if (s == 0) stage_slab_relu<0, kGate>(acc, slab, row, ok[0], ok[1], lane);
            else stage_slab_relu<(kBN64 > 1 ? 1 : 0), kGate>(acc, slab, row, ok[0], ok[1], lane);
          } else {
            if (s == 0) stage_slab<0>(acc, slab, row, ok[0], ok[1], lane);
            else stage_slab<(kBN64 > 1 ? 1 : 0)>(acc, slab, row, ok[0], ok[1], lane);
          }
          fence_proxy_async_smem();
          named_bar_sync(1, kConsumerThreads);
          if (issuer) {
            tma_store_4d(&omap, slab, co0, tw * p.bw, th * p.bh, tn * p.bn);
            tma_store_commit();
          }
          if (bn_row && wg == 0) slab_bn_stats(slab, cw, lane, bn_row, co0, p.N);   // next to the bulk store's own read
          ++slab_ctr;
        }
      } else {
        // direct global stores (fp32 output / bias: the dense layer)
#pragma unroll
        for (int jc = 0; jc < BN / 8; ++jc) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int co = n_tile * BN + 8 * jc + 2 * (lane & 3) + e;
              if (ok[h] && co < p.N) {
                float a = acc[4 * jc + 2 * h + e];
                if (p.bias) a += __ldg(p.bias + co);
                if (p.out_bf16) p.out_bf16[o_pix[h] + co] = __float2bfloat16(a);
                if (p.out_f32) p.out_f32[o_pix[h] + co] = a;
              }
            }
          }
        }
      }
    }
    if (p.tma_store && issuer) tma_store_wait_all();   // smem must outlive the bulk stores
  }
}

template <int BN, int STAGES>
__global__ void __launch_bounds__(kThreads, 1)
k_igemm_kmajor(const __grid_constant__ TMaps4 amaps, const __grid_constant__ CUtensorMap bmap,
               const __grid_constant__ CUtensorMap omap, const IgemmParams p) {
  kmajor_body<BN, STAGES, kEpiPlain>(amaps, bmap, omap, p, nullptr, BnEpilogue{});
}

// fprop with the inference batch norm in the epilogue (rmap: the residual, same layout as the output; unused
// without ep.residual).  Requires p.tma_store.
template <int BN, int STAGES>
__global__ void __launch_bounds__(kThreads, 1)
k_igemm_kmajor_bn(const __grid_constant__ TMaps4 amaps, const __grid_constant__ CUtensorMap bmap,
                  const __grid_constant__ CUtensorMap omap, const IgemmParams p,
                  const __grid_constant__ CUtensorMap rmap, const BnEpilogue ep) {
  kmajor_body<BN, STAGES, kEpiBn>(amaps, bmap, omap, p, &rmap, ep);
}

// fprop with the ReLU in the epilogue (kGate false; rmap unused), or the dgrad gated by the layer's forward input
// x > 0 (kGate true; rmap: x through dx's view, same boxes and swizzle as the store).  Requires p.tma_store.
template <int BN, int STAGES, bool kGate>
__global__ void __launch_bounds__(kThreads, 1)
k_igemm_kmajor_relu(const __grid_constant__ TMaps4 amaps, const __grid_constant__ CUtensorMap bmap,
                    const __grid_constant__ CUtensorMap omap, const IgemmParams p,
                    const __grid_constant__ CUtensorMap rmap) {
  kmajor_body<BN, STAGES, kGate ? kEpiReluGate : kEpiRelu>(amaps, bmap, omap, p, &rmap, BnEpilogue{});
}

// ----------------------------------------------------------------------------
// wgrad kernel: D[128 ci, BN co] += X^T[ci, 64 pix] * dY[64 pix, co]  (both MN-major)
// ----------------------------------------------------------------------------
struct WgradParams {
  int ntaps;
  TapInfo taps[kMaxTaps];
  int GW, GH, NB;                   // output pixel grid (the reduction domain)
  int bw, bh, bn;                   // pixel box of one K block (bw*bh*bn == 64)
  int tiles_w, tiles_h, tiles_n;
  int pblocks, splits, pblocks_per_split;
  int ci, co;                       // M and N extents
  int m_tiles, n_tiles;
  float* out;                       // [splits][taps][ci][co] partials (or dw itself when splits == 1)
  long long split_stride;           // elements between split slices
};

// Same warp roles as k_igemm_kmajor; consumer warpgroup w owns input channels 64w..64w+63 of the unit (the
// w-th 64-channel x box of a stage is its whole A operand).
template <int BN, int STAGES>
__global__ void __launch_bounds__(kThreads, 1)
k_igemm_wgrad(const __grid_constant__ TMaps4 xmaps, const __grid_constant__ CUtensorMap dymap,
              const WgradParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  constexpr uint32_t kABytes = kBM * kBK * 2;        // two 64-channel boxes of 64 pixels: 16 KB
  constexpr uint32_t kBBytes = BN * kBK * 2;
  constexpr uint32_t kStageBytes = kABytes + kBBytes;
  constexpr uint32_t kBox = 64 * 64 * 2;             // 8 KB: 64 pixels x 64 channels
  constexpr int kBBoxes = BN / 64;

  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_base = smem_base + STAGES * kStageBytes;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < 4; ++i) prefetch_tmap(&xmaps.a[i]);
    prefetch_tmap(&dymap);
    for (int s = 0; s < STAGES; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), kConsumerWarps); }
    fence_barrier_init();
  }
  __syncthreads();

  // Work units: (split, N tile, M index) with M index = tap * m_tiles + m_tile, dealt round-robin to CTAs.
  // `live` (mi < mcount) always holds; the guarded selects below are kept because nvcc cannot prove it, and dropping
  // them reschedules the main loop around the wgmma.
  const int mcount = p.ntaps * p.m_tiles;
  const int units_per_split = mcount * p.n_tiles;
  const int total_units = units_per_split * p.splits;
  const int first = blockIdx.x, step = gridDim.x;

  if (warp == 0) {
    int stage = 0; uint32_t phase = 0;                     // converged warp, one elected lane issues
    for (int q = first; q < total_units; q += step) {
      const int split = q / units_per_split;
      const int r = q % units_per_split;
      const int n_tile = r % p.n_tiles;
      const int mi = r / p.n_tiles;
      const bool live = mi < mcount;
      const TapInfo tap = p.taps[live ? mi / p.m_tiles : 0];
      const int c_base = live ? (mi % p.m_tiles) * kBM : (1 << 28);
      const int pb0 = split * p.pblocks_per_split;
      const int pb1 = min(pb0 + p.pblocks_per_split, p.pblocks);
      int tw = pb0 % p.tiles_w, th = (pb0 / p.tiles_w) % p.tiles_h, tn = pb0 / (p.tiles_w * p.tiles_h);
      for (int pb = pb0; pb < pb1; ++pb) {
        mbar_wait(empty_bar(stage), phase ^ 1u);
        if (elect_one()) {
          const uint32_t a_dst = smem_base + stage * kStageBytes;
          const uint32_t b_dst = a_dst + kABytes;
          mbar_arrive_expect_tx(full_bar(stage), kStageBytes);
#pragma unroll
          for (int h = 0; h < kBM / 64; ++h)
            tma_load_4d(a_dst + h * kBox, &xmaps.a[tap.map_id], full_bar(stage), c_base + h * 64,
                        tw * p.bw + tap.dw, th * p.bh + tap.dh, tn * p.bn);
#pragma unroll
          for (int h = 0; h < kBBoxes; ++h)
            tma_load_4d(b_dst + h * kBox, &dymap, full_bar(stage), n_tile * BN + h * 64, tw * p.bw,
                        th * p.bh, tn * p.bn);
        }
        __syncwarp();
        if (++tw == p.tiles_w) { tw = 0; if (++th == p.tiles_h) { th = 0; ++tn; } }   // next pixel block (no divisions)
        if (++stage == STAGES) { stage = 0; phase ^= 1u; }
      }
    }
  } else if (warp >= kConsumerWarp0) {
    const int cw = warp - kConsumerWarp0;
    const int wg = cw >> 2;
    const int row = 64 * wg + 16 * (cw & 3) + (lane >> 2);
    float acc[BN / 2];
    int stage = 0; uint32_t phase = 0;
    for (int q = first; q < total_units; q += step) {
      const int split = q / units_per_split;
      const int r = q % units_per_split;
      const int n_tile = r % p.n_tiles;
      const int mi = r / p.n_tiles;
      const bool live = mi < mcount;
      const int tap_idx = live ? mi / p.m_tiles : 0;
      const int pb0 = split * p.pblocks_per_split;
      const int pb1 = min(pb0 + p.pblocks_per_split, p.pblocks);
      zero_acc(acc);
      int prev = -1;
      for (int pb = pb0; pb < pb1; ++pb) {
        mbar_wait(full_bar(stage), phase);
        const uint32_t a_src = smem_base + stage * kStageBytes;
        const uint64_t da = make_smem_desc(a_src + (uint32_t)wg * kBox, kBox, 1024);
        const uint64_t db = make_smem_desc(a_src + kABytes, kBox, 1024);
        fence_regs(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBK / 16; ++k)              // 16 pixels = 16 rows of 128 B = +128 address units
          Wgmma<BN>::template ss<1, 1>(acc, da + 128 * k, db + 128 * k);
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0 && lane == 0) mbar_arrive(empty_bar(prev));
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1u; }
      }
      wgmma_wait<0>();
      fence_regs(acc);
      if (prev >= 0 && lane == 0) mbar_arrive(empty_bar(prev));

      const int m0 = live ? (mi % p.m_tiles) * kBM : p.ci;
      float* base = p.out + (long long)split * p.split_stride + (long long)p.taps[tap_idx].b_tap * p.ci * p.co;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int ci = m0 + row + 8 * h;
        if (ci >= p.ci) continue;
#pragma unroll
        for (int jc = 0; jc < BN / 8; ++jc) {
          const int co = n_tile * BN + 8 * jc + 2 * (lane & 3);          // co is even and p.co % 8 == 0
          if (co < p.co)
            *reinterpret_cast<float2*>(base + (long long)ci * p.co + co) =
                make_float2(acc[4 * jc + 2 * h], acc[4 * jc + 2 * h + 1]);
        }
      }
    }
  }
}

// dw = beta * dw + sum_s partial[s]   (fixed summation order => deterministic)
__global__ void k_splitk_reduce(const float* __restrict__ part, long long split_stride, int splits,
                                float* __restrict__ dw, long long n, float beta) {
  const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (i >= n) return;
  if (i + 3 < n) {
    float4 acc = beta != 0.f ? *reinterpret_cast<const float4*>(dw + i) : make_float4(0.f, 0.f, 0.f, 0.f);
    for (int s = 0; s < splits; ++s) {
      const float4 v = *reinterpret_cast<const float4*>(part + (long long)s * split_stride + i);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    *reinterpret_cast<float4*>(dw + i) = acc;
  } else {
    for (long long j = i; j < n; ++j) {
      float a = beta != 0.f ? dw[j] : 0.f;
      for (int s = 0; s < splits; ++s) a += part[(long long)s * split_stride + j];
      dw[j] = a;
    }
  }
}

// ----------------------------------------------------------------------------
// Host side
// ----------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn g_encode = nullptr;
static bool g_bn_stats_always = false;   // rigl_set_bn_stats_always: epilogue statistics for every supported shape (tests)
static int g_num_sms = 0;
static std::once_flag g_once;
static int g_init_status = RIGL_OK;

static void init_driver() {
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
  if (e != cudaSuccess || fn == nullptr || qres != cudaDriverEntryPointSuccess) {
    set_error("cuTensorMapEncodeTiled not available from the driver (%s)", cudaGetErrorString(e));
    g_init_status = RIGL_ERR_DRIVER;
    return;
  }
  g_encode = reinterpret_cast<EncodeTiledFn>(fn);
  int dev = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
  if (g_num_sms <= 0) g_num_sms = kNumSmsHint;
}

static int ensure_driver() {
  // The driver entry point needs a CUDA context current on THIS thread (autograd runs
  // backward on worker threads that may not have touched the runtime yet).
  static thread_local bool ctx_ready = false;
  if (!ctx_ready) {
    cudaFree(0);
    ctx_ready = true;
  }
  std::call_once(g_once, init_driver);
  return g_init_status;
}

// RIGL_HALO3X3=0: 3x3/s1 layers with <= 64 channels use the generic kernels.
static bool halo_enabled() {
  static const bool on = [] {
    const char* e = getenv("RIGL_HALO3X3");
    return !(e && e[0] == '0');
  }();
  return on;
}

// Raises kernel K's dynamic shared-memory limit to `smem` bytes the first time a launch needs that much.  The limit
// only grows, so a smaller launch after a larger one makes no call.
template <auto K>
static cudaError_t smem_limit(size_t smem) {
  static size_t configured = 0;
  if (smem <= configured) return cudaSuccess;
  const cudaError_t e = cudaFuncSetAttribute(K, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e == cudaSuccess) configured = smem;
  return e;
}

// bf16 tensor map over `rank` dims (dim 0 innermost, contiguous), 128B swizzle, zero OOB fill.
static int make_tmap_swz(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                         const uint64_t* strides_bytes /*rank-1*/, const uint32_t* box, CUtensorMapSwizzle swz) {
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  cuuint64_t gdim[5], gstr[4];
  cuuint32_t bx[5];
  for (int i = 0; i < rank; ++i) { gdim[i] = dims[i]; bx[i] = box[i]; }
  for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
  CUresult r = g_encode(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base), gdim,
                        gstr, bx, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d): rank %d dims [%llu,%llu,%llu,%llu] box [%u,%u,%u,%u]", (int)r,
              rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
              (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 3 ? dims[3] : 0), box[0],
              rank > 1 ? box[1] : 0, rank > 2 ? box[2] : 0, rank > 3 ? box[3] : 0);
    return RIGL_ERR_DRIVER;
  }
  return RIGL_OK;
}
static int make_tmap(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                     const uint64_t* strides_bytes /*rank-1*/, const uint32_t* box) {
  return make_tmap_swz(out, base, rank, dims, strides_bytes, box, CU_TENSOR_MAP_SWIZZLE_128B);
}

// Activation view (C, W_r, H_r, N) of an NHWC tensor sub-sampled by `s` at parity (rh, rw).
static int make_act_map(CUtensorMap* out, const void* base, int nb, int h, int w, int c, int pitch, int s, int rh,
                        int rw, const uint32_t box[4]) {
  const uint64_t hr = (h - rh + s - 1) / s, wr = (w - rw + s - 1) / s;
  const uint64_t dims[4] = {(uint64_t)c, wr, hr, (uint64_t)nb};
  const uint64_t strides[3] = {(uint64_t)s * pitch * 2, (uint64_t)s * w * pitch * 2, (uint64_t)h * w * pitch * 2};
  const uint8_t* p = static_cast<const uint8_t*>(base) + ((size_t)rh * w + rw) * pitch * 2;
  return make_tmap(out, p, 4, dims, strides, box);
}

// Smallest-waste factorisation bw*bh*bn == total (powers of two) for a GW x GH x NB pixel grid.
static void choose_box(int gw, int gh, int nb, int total, int* bw, int* bh, int* bn) {
  long long best = -1;
  for (int w = 1; w <= total; w *= 2)
    for (int h = 1; w * h <= total; h *= 2) {
      const int n = total / (w * h);
      const long long padded = (long long)((gw + w - 1) / w * w) * ((gh + h - 1) / h * h) * ((nb + n - 1) / n * n);
      // prefer less padding; then longer contiguous runs (larger w, then larger h)
      const long long score = padded * 1024 - w * 16 - h;
      if (best < 0 || score < best) { best = score; *bw = w; *bh = h; *bn = n; }
    }
}

static inline int floordiv(int a, int b) { return (a >= 0) ? a / b : -((-a + b - 1) / b); }
static inline int posmod(int a, int b) { return ((a % b) + b) % b; }

// Tiling of a launch's gw x gh x nb pixel grid by boxes of `box_pixels` pixels (IgemmParams or WgradParams).
template <typename P>
static void set_pixel_tiling(P& p, int gw, int gh, int nb, int box_pixels) {
  p.GW = gw; p.GH = gh; p.NB = nb;
  choose_box(gw, gh, nb, box_pixels, &p.bw, &p.bh, &p.bn);
  p.tiles_w = (gw + p.bw - 1) / p.bw; p.tiles_h = (gh + p.bh - 1) / p.bh; p.tiles_n = (nb + p.bn - 1) / p.bn;
}

// Every filter tap of g reads x at its output pixels shifted by the tap offset.  With stride s, x is viewed through
// one parity sub-grid map per (kh - pad, kw - pad) mod s (up to four); maps no tap uses alias a used one.
template <typename P>
static int set_conv_taps(P& p, TMaps4* maps, const ConvGeom& g, const void* x, const uint32_t box[4]) {
  bool made[4] = {false, false, false, false};
  p.ntaps = 0;
  for (int kh = 0; kh < g.ksize; ++kh)
    for (int kw = 0; kw < g.ksize; ++kw) {
      const int rh = posmod(kh - g.pad, g.stride), rw = posmod(kw - g.pad, g.stride);
      const int id = rh * g.stride + rw;
      if (!made[id]) {
        const int rc = make_act_map(&maps->a[id], x, g.batch, g.in_h, g.in_w, g.cin, g.x_pitch, g.stride, rh, rw, box);
        if (rc != RIGL_OK) return rc;
        made[id] = true;
      }
      TapInfo& t = p.taps[p.ntaps++];
      t.map_id = (int8_t)id; t.dh = (int8_t)floordiv(kh - g.pad, g.stride); t.dw = (int8_t)floordiv(kw - g.pad, g.stride);
      t.b_tap = kh * g.ksize + kw;
    }
  for (int i = 0; i < 4; ++i) if (!made[i]) maps->a[i] = maps->a[p.taps[0].map_id];
  return RIGL_OK;
}

int tc_max_ctas() {
  ensure_driver();
  return g_num_sms > 0 ? g_num_sms : kNumSmsHint;
}

bool tc_supported(const ConvGeom& g, int which) {
  if (g.x_pitch % 8 || g.cout % 8) return false;     // 16-byte row pitches for TMA
  if (which == 1 && g.cin % 8) return false;         // dgrad stores 8 channels at a time
  if (g.stride != 1 && g.stride != 2) return false;
  if (g.ksize * g.ksize > kMaxTaps) return false;
  (void)which;
  return true;
}

static size_t wgrad_ws_elems(const ConvGeom& g, int* splits_out, int* bps_out, int bw, int bh, int bn, int bn_tile) {
  const int tiles_w = (g.out_w + bw - 1) / bw, tiles_h = (g.out_h + bh - 1) / bh, tiles_n = (g.batch + bn - 1) / bn;
  const int pblocks = tiles_w * tiles_h * tiles_n;
  const int out_tiles = g.taps() * ((g.cin + kBM - 1) / kBM) * ((g.cout + bn_tile - 1) / bn_tile);
  const int sms = g_num_sms > 0 ? g_num_sms : kNumSmsHint;
  int splits = (2 * sms + out_tiles - 1) / out_tiles;
  if (splits > pblocks) splits = pblocks;
  if (splits < 1) splits = 1;
  const int bps = (pblocks + splits - 1) / splits;
  splits = (pblocks + bps - 1) / bps;
  if (splits_out) *splits_out = splits;
  if (bps_out) *bps_out = bps;
  return (size_t)splits * g.taps() * g.cin * g.cout;
}

// Wider N tiles halve the L2->smem bytes per FLOP (the wgrad main loop is L2-bandwidth bound: K blocks are
// only 64 pixels deep); 128 is the widest whose accumulators fit the consumer warpgroups' registers.
static int wgrad_bn_tile(const ConvGeom& g) { return g.cout >= 128 ? 128 : 64; }

#include "halo3x3.cuh"
#include "stem_s2d.cuh"

size_t tc_workspace_bytes(const ConvGeom& g) {
  if (!tc_supported(g, 2)) return 0;
  int bw, bh, bn;
  choose_box(g.out_w, g.out_h, g.batch, 64, &bw, &bh, &bn);
  size_t elems = wgrad_ws_elems(g, nullptr, nullptr, bw, bh, bn, wgrad_bn_tile(g));
  HaloParams hp;
  if (halo_wgrad_ok(g, &hp)) { const size_t e = halo_wgrad_ws_elems(g, hp); if (e > elems) elems = e; }
  return elems * sizeof(float) + 256;
}

int conv_route(const ConvGeom& g, int which, const ConvEpilogue& epi) {
  static const char* const kName[] = {"plain", "fused BN statistics", "fused BN apply", "fused ReLU", "gated dgrad"};
  const char* name = kName[epi.kind];
  if (force_simt() || !tc_supported(g, which)) {
    if (epi.kind == ConvEpilogue::kPlain) return kPathSimt;
    set_error("%s: shape not on the tensor-core kernels", name);
    return RIGL_ERR_UNSUPPORTED;
  }
  if (epi.kind == ConvEpilogue::kReluGate && g.stride != 1) {   // the strided dgrad is one launch per parity class
    set_error("%s: shape has no gated dgrad (stride %d)", name, g.stride);
    return RIGL_ERR_UNSUPPORTED;
  }
  HaloParams hp;
  const bool halo = which == 0   ? epi.out_f32 == nullptr && epi.bias == nullptr && halo_fprop_ok(g, &hp)
                    : which == 1 ? halo_dgrad_ok(g, &hp)
                                 : halo_wgrad_ok(g, &hp);
  if (halo) {
    if (epi.kind == ConvEpilogue::kPlain || epi.kind == ConvEpilogue::kRelu) return kPathHalo;
    set_error("%s: layer runs on the halo kernels", name);   // the caller runs the plain call + the separate pass
    return RIGL_ERR_UNSUPPORTED;
  }
  if (epi.kind == ConvEpilogue::kBnStats && !g_bn_stats_always) {
    // The statistics are free when the tile's main loop is long enough to hide them (reduction length
    // K = taps * cin >= 512), and cost about what the separate stats pass costs -- or more -- for the short-K /
    // wide-output layers whose epilogue is the bottleneck (1x1 convs with K <= 128; K = 256 with more than 128
    // output channels).
    const int K = g.taps() * g.cin;
    if (!(K >= 512 || (K >= 256 && g.cout <= 128))) {
      set_error("%s: not profitable for this shape (K = %d, cout = %d)", name, K, g.cout);
      return RIGL_ERR_UNSUPPORTED;
    }
  }
  return kPathKmajor;
}

static int kmajor_grid(const IgemmParams& p) {         // CTAs the K-major launcher will use (p.n_tiles set)
  const int tiles = p.tiles_w * p.tiles_h * p.tiles_n * p.n_tiles;
  return tiles < g_num_sms ? tiles : g_num_sms;
}

// The K-major kernel with epi's epilogue: k_igemm_kmajor (kPlain; kBnStats through p.bn_partial), k_igemm_kmajor_bn
// (kBnApply, residual map rmap) or k_igemm_kmajor_relu (kRelu; kReluGate with the gate map rmap).  Variants that read
// no second tensor get the output map as rmap.
template <int BN, int STAGES>
static int launch_kmajor(const TMaps4& amaps, const CUtensorMap& bmap, const CUtensorMap& omap, const IgemmParams& p,
                         const ConvEpilogue& epi, const CUtensorMap& rmap, cudaStream_t s) {
  // (the 256 bytes past the slabs hold the 2 * STAGES ring barriers and the residual barrier)
  constexpr size_t smem = (size_t)STAGES * (kBM * kBK * 2 + BN * kBK * 2) + 2 * (kBM * 64 * 2) + 1024 + 256;
  static_assert(smem <= 227 * 1024, "K-major kernel exceeds the shared memory of an SM");
  static_assert(8 * (2 * STAGES + 1) <= 256, "K-major kernel barriers exceed their shared memory");
  const int grid = kmajor_grid(p);
  const char* name;
  switch (epi.kind) {
    case ConvEpilogue::kBnApply: {
      const BnEpilogue ep = {epi.scale, epi.shift, epi.relu ? 1 : 0, epi.residual ? 1 : 0};
      RIGL_CUDA(smem_limit<k_igemm_kmajor_bn<BN, STAGES>>(smem));
      k_igemm_kmajor_bn<BN, STAGES><<<grid, kThreads, smem, s>>>(amaps, bmap, omap, p, rmap, ep);
      name = "k_igemm_kmajor_bn";
      break;
    }
    case ConvEpilogue::kRelu:
      RIGL_CUDA(smem_limit<k_igemm_kmajor_relu<BN, STAGES, false>>(smem));
      k_igemm_kmajor_relu<BN, STAGES, false><<<grid, kThreads, smem, s>>>(amaps, bmap, omap, p, rmap);
      name = "k_igemm_kmajor_relu";
      break;
    case ConvEpilogue::kReluGate:
      RIGL_CUDA(smem_limit<k_igemm_kmajor_relu<BN, STAGES, true>>(smem));
      k_igemm_kmajor_relu<BN, STAGES, true><<<grid, kThreads, smem, s>>>(amaps, bmap, omap, p, rmap);
      name = "k_igemm_kmajor_relu";
      break;
    default:
      RIGL_CUDA(smem_limit<k_igemm_kmajor<BN, STAGES>>(smem));
      k_igemm_kmajor<BN, STAGES><<<grid, kThreads, smem, s>>>(amaps, bmap, omap, p);
      name = "k_igemm_kmajor";
  }
  RIGL_LAUNCH_CHECK(name);
  return RIGL_OK;
}

static int dispatch_kmajor(int n_out, const TMaps4& amaps, const CUtensorMap& bmap, const CUtensorMap& omap,
                           IgemmParams& p, int bn_tile, const ConvEpilogue& epi, const CUtensorMap& rmap,
                           cudaStream_t s) {
  p.n_tiles = (n_out + bn_tile - 1) / bn_tile;
  if (bn_tile == 64) return launch_kmajor<64, 7>(amaps, bmap, omap, p, epi, rmap, s);
  return launch_kmajor<128, 5>(amaps, bmap, omap, p, epi, rmap, s);
}

static int pick_bn(int n_out) {
  // The widest tile whose accumulators fit the consumer warpgroups' registers (64 x 128 fp32 per warpgroup):
  // fewest A re-reads.
  return n_out > 64 ? 128 : 64;
}

void tc_set_bn_stats_always(bool on) { g_bn_stats_always = on; }

int tc_fprop(const ConvGeom& g, int path, const void* x, const void* packed, void* y, const ConvEpilogue& epi,
             cudaStream_t s) {
  int rc = ensure_driver();
  if (rc != RIGL_OK) return rc;
  const PackedLayout L = packed_layout(g.taps(), g.cin, g.cout);
  const uint8_t* pk = static_cast<const uint8_t*>(packed);
  if (path == kPathHalo) {
    HaloParams hp = {};
    halo_fprop_ok(g, &hp);            // (true: conv_route chose the halo kernels)
    return halo_launch_kmajor(hp, x, g.cin, g.x_pitch, pk + L.off_fprop, L.cin_pad, g.cout, y, g.cout, false, s,
                              epi.kind == ConvEpilogue::kRelu);
  }
  IgemmParams p = {};
  set_pixel_tiling(p, g.out_w, g.out_h, g.batch, 128);
  p.kblks = (g.cin + kBK - 1) / kBK;
  p.N = g.cout;
  p.out_bf16 = static_cast<__nv_bfloat16*>(y); p.out_f32 = epi.out_f32; p.bias = epi.bias;
  p.o_off = 0; p.o_sw = g.cout; p.o_sh = (long long)g.out_w * g.cout; p.o_sn = (long long)g.out_h * g.out_w * g.cout;
  p.nnz = reinterpret_cast<const uint32_t*>(pk + L.off_nnz);
  p.nnz_tap_stride = L.n_tiles * L.k_tiles; p.nnz_n_stride = L.k_tiles; p.nnz_k_stride = 1;
  p.bn_partial = epi.bn_partial;
  TMaps4 amaps;
  const uint32_t abox[4] = {(uint32_t)kBK, (uint32_t)p.bw, (uint32_t)p.bh, (uint32_t)p.bn};
  rc = set_conv_taps(p, &amaps, g, x, abox);
  if (rc != RIGL_OK) return rc;
  const int bn_tile = pick_bn(g.cout);
  CUtensorMap bmap;
  const uint64_t bdims[3] = {(uint64_t)L.cin_pad, (uint64_t)g.cout, (uint64_t)g.taps()};
  const uint64_t bstr[2] = {(uint64_t)L.cin_pad * 2, (uint64_t)g.cout * L.cin_pad * 2};
  const uint32_t bbox[3] = {(uint32_t)kBK, (uint32_t)bn_tile, 1};
  rc = make_tmap(&bmap, pk + L.off_fprop, 3, bdims, bstr, bbox);
  if (rc != RIGL_OK) return rc;
  CUtensorMap omap = bmap;
  p.tma_store = (y != nullptr && epi.out_f32 == nullptr && epi.bias == nullptr) ? 1 : 0;
  if (p.tma_store) {
    rc = make_act_map(&omap, y, g.batch, g.out_h, g.out_w, g.cout, g.cout, 1, 0, 0, abox);
    if (rc != RIGL_OK) return rc;
  }
  if (epi.kind == ConvEpilogue::kBnStats && epi.bn_rows) {
    p.n_tiles = (g.cout + bn_tile - 1) / bn_tile;
    *epi.bn_rows = kmajor_grid(p);
  }
  CUtensorMap rmap = omap;
  if (epi.kind == ConvEpilogue::kBnApply && epi.residual) {   // the residual through the output's view
    rc = make_act_map(&rmap, epi.residual, g.batch, g.out_h, g.out_w, g.cout, g.cout, 1, 0, 0, abox);
    if (rc != RIGL_OK) return rc;
  }
  return dispatch_kmajor(g.cout, amaps, bmap, omap, p, bn_tile, epi, rmap, s);
}

int tc_dgrad(const ConvGeom& g, int path, const void* dy, const void* packed, void* dx, const ConvEpilogue& epi,
             cudaStream_t s) {
  int rc = ensure_driver();
  if (rc != RIGL_OK) return rc;
  const PackedLayout L = packed_layout(g.taps(), g.cin, g.cout);
  const uint8_t* pk = static_cast<const uint8_t*>(packed);
  const int st = g.stride;
  if (path == kPathHalo) {
    HaloParams hp = {};
    halo_dgrad_ok(g, &hp);            // (true: conv_route chose the halo kernels)
    return halo_launch_kmajor(hp, dy, g.cout, g.cout, pk + L.off_dgrad, L.cout_pad, g.cin, dx, g.x_pitch, true, s);
  }
  // classes of input pixels by parity; each class is one launch over its sub-grid
  bool need_zero = false;
  for (int ph = 0; ph < st && !need_zero; ++ph)
    for (int pw = 0; pw < st; ++pw) {
      int n = 0;
      for (int kh = 0; kh < g.ksize; ++kh)
        for (int kw = 0; kw < g.ksize; ++kw)
          if (posmod(ph + g.pad - kh, st) == 0 && posmod(pw + g.pad - kw, st) == 0) ++n;
      if (n == 0) need_zero = true;
    }
  if (need_zero) RIGL_CUDA(cudaMemsetAsync(dx, 0, (size_t)g.in_pixels() * g.x_pitch * 2, s));
  for (int ph = 0; ph < st; ++ph)
    for (int pw = 0; pw < st; ++pw) {
      IgemmParams p = {};
      const int gh = (g.in_h - ph + st - 1) / st, gw = (g.in_w - pw + st - 1) / st;
      if (gh <= 0 || gw <= 0) continue;
      p.ntaps = 0;
      for (int kh = 0; kh < g.ksize; ++kh)
        for (int kw = 0; kw < g.ksize; ++kw)
          if (posmod(ph + g.pad - kh, st) == 0 && posmod(pw + g.pad - kw, st) == 0) {
            TapInfo& t = p.taps[p.ntaps++];
            t.map_id = 0; t.dh = (int8_t)((ph + g.pad - kh) / st); t.dw = (int8_t)((pw + g.pad - kw) / st);
            t.b_tap = kh * g.ksize + kw;
          }
      if (p.ntaps == 0) continue;
      set_pixel_tiling(p, gw, gh, g.batch, 128);
      p.kblks = (g.cout + kBK - 1) / kBK;
      p.N = g.cin;
      // survivor table indexed [tap][co/64][ci/64]: here N = ci, K = co
      p.nnz = reinterpret_cast<const uint32_t*>(pk + L.off_nnz);
      p.nnz_tap_stride = L.n_tiles * L.k_tiles; p.nnz_n_stride = 1; p.nnz_k_stride = L.k_tiles;
      TMaps4 amaps;
      const uint32_t abox[4] = {(uint32_t)kBK, (uint32_t)p.bw, (uint32_t)p.bh, (uint32_t)p.bn};
      rc = make_act_map(&amaps.a[0], dy, g.batch, g.out_h, g.out_w, g.cout, g.cout, 1, 0, 0, abox);
      if (rc != RIGL_OK) return rc;
      for (int i = 1; i < 4; ++i) amaps.a[i] = amaps.a[0];
      const int bn_tile = pick_bn(g.cin);
      CUtensorMap bmap;
      const uint64_t bdims[3] = {(uint64_t)L.cout_pad, (uint64_t)g.cin, (uint64_t)g.taps()};
      const uint64_t bstr[2] = {(uint64_t)L.cout_pad * 2, (uint64_t)g.cin * L.cout_pad * 2};
      const uint32_t bbox[3] = {(uint32_t)kBK, (uint32_t)bn_tile, 1};
      rc = make_tmap(&bmap, pk + L.off_dgrad, 3, bdims, bstr, bbox);
      if (rc != RIGL_OK) return rc;
      CUtensorMap omap;                  // dx viewed through the parity sub-grid of this launch
      rc = make_act_map(&omap, dx, g.batch, g.in_h, g.in_w, g.cin, g.x_pitch, st, ph, pw, abox);
      if (rc != RIGL_OK) return rc;
      p.tma_store = 1;
      CUtensorMap rmap = omap;
      if (epi.kind == ConvEpilogue::kReluGate) {   // x through dx's view: the gate box is the output box
        rc = make_act_map(&rmap, epi.gate, g.batch, g.in_h, g.in_w, g.cin, g.x_pitch, st, ph, pw, abox);
        if (rc != RIGL_OK) return rc;
      }
      rc = dispatch_kmajor(g.cin, amaps, bmap, omap, p, bn_tile, epi, rmap, s);
      if (rc != RIGL_OK) return rc;
    }
  return RIGL_OK;
}

template <int BN, int STAGES>
static int launch_wgrad(const TMaps4& xmaps, const CUtensorMap& dymap, const WgradParams& p, cudaStream_t s) {
  constexpr size_t smem = (size_t)STAGES * (kBM * kBK * 2 + BN * kBK * 2) + 1024 + 256;
  static_assert(smem <= 227 * 1024, "wgrad kernel exceeds the shared memory of an SM");
  RIGL_CUDA(smem_limit<k_igemm_wgrad<BN, STAGES>>(smem));
  const int units = p.ntaps * p.m_tiles * p.n_tiles * p.splits;
  const int grid = units < g_num_sms ? units : g_num_sms;
  k_igemm_wgrad<BN, STAGES><<<grid, kThreads, smem, s>>>(xmaps, dymap, p);
  RIGL_LAUNCH_CHECK("k_igemm_wgrad");
  return RIGL_OK;
}

int tc_wgrad(const ConvGeom& g, int path, const void* x, const void* dy, float* dw, float beta, void* ws,
             size_t ws_bytes, cudaStream_t s) {
  int rc = ensure_driver();
  if (rc != RIGL_OK) return rc;
  if (path == kPathHalo) {
    HaloParams hp = {};
    halo_wgrad_ok(g, &hp);            // (true: conv_route chose the halo kernels)
    const size_t need = halo_wgrad_ws_elems(g, hp) * sizeof(float);
    float* wsf = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(ws) + 255) & ~(uintptr_t)255);
    if (ws == nullptr || ws_bytes < need + 256) {
      set_error("rigl_conv2d_wgrad_dense: workspace %zu < required %zu", ws_bytes, need + 256);
      return RIGL_ERR_WORKSPACE;
    }
    rc = halo_launch_wgrad(hp, g, x, dy, wsf, s);
    if (rc != RIGL_OK) return rc;
    const long long n_w9 = (long long)9 * g.cin * g.cout;
    const long long threads = (n_w9 + 3) / 4;
    k_splitk_reduce<<<(unsigned)((threads + 255) / 256), 256, 0, s>>>(wsf, n_w9, halo_wgrad_grid(hp), dw, n_w9, beta);
    RIGL_LAUNCH_CHECK("k_splitk_reduce");
    return RIGL_OK;
  }
  WgradParams p = {};
  set_pixel_tiling(p, g.out_w, g.out_h, g.batch, 64);
  p.pblocks = p.tiles_w * p.tiles_h * p.tiles_n;
  const int bn_tile = wgrad_bn_tile(g);
  const size_t elems = wgrad_ws_elems(g, &p.splits, &p.pblocks_per_split, p.bw, p.bh, p.bn, bn_tile);
  p.ci = g.cin; p.co = g.cout;
  p.m_tiles = (g.cin + kBM - 1) / kBM; p.n_tiles = (g.cout + bn_tile - 1) / bn_tile;
  const long long n_w = (long long)g.taps() * g.cin * g.cout;
  const bool direct = (p.splits == 1 && beta == 0.f);
  if (!direct) {
    const size_t need = elems * sizeof(float);
    if (ws == nullptr || ws_bytes < need + 256) {
      set_error("rigl_conv2d_wgrad_dense: workspace %zu < required %zu", ws_bytes, need + 256);
      return RIGL_ERR_WORKSPACE;
    }
    p.out = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(ws) + 255) & ~(uintptr_t)255);
    p.split_stride = n_w;
  } else {
    p.out = dw; p.split_stride = 0;
  }
  TMaps4 xmaps;
  const uint32_t box[4] = {64, (uint32_t)p.bw, (uint32_t)p.bh, (uint32_t)p.bn};
  rc = set_conv_taps(p, &xmaps, g, x, box);
  if (rc != RIGL_OK) return rc;
  CUtensorMap dymap;
  rc = make_act_map(&dymap, dy, g.batch, g.out_h, g.out_w, g.cout, g.cout, 1, 0, 0, box);
  if (rc != RIGL_OK) return rc;
  rc = (bn_tile == 128) ? launch_wgrad<128, 6>(xmaps, dymap, p, s) : launch_wgrad<64, 8>(xmaps, dymap, p, s);
  if (rc != RIGL_OK) return rc;
  if (!direct) {
    const long long threads = (n_w + 3) / 4;
    k_splitk_reduce<<<(unsigned)((threads + 255) / 256), 256, 0, s>>>(p.out, p.split_stride, p.splits, dw, n_w, beta);
    RIGL_LAUNCH_CHECK("k_splitk_reduce");
  }
  return RIGL_OK;
}

}  // namespace rigl
