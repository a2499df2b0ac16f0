// Batched RigL/SET mask update on sm_90a: exact top-k drop by |mask*w| (+noise)
// and exact top-k grow by |dense grad| with tf.nn.top_k tie semantics
// (equal scores -> lower flat index first), for ALL masked layers of a model in
// one 7-node launch sequence, masks stored as 1-bit bitmaps.
//
// Replaces sparse_optimizers_base.py:276-343 (_get_update_op) and its callers'
// score construction (:260-274, :523-538), grow init (:355-400, :540-553) and
// slot reset (:345-353, :555-564).  The reference does two full sorts of every
// layer; here each selection is a radix SELECT:
//   A  k_hist_drop   : 4096-bin histogram of the top 12 bits of the order-
//                      preserving key of score_drop, all layers, one launch
//   B  k_pick_drop   : per layer: popcount -> n_ones, n_prune, n_keep; find the
//                      threshold bin
//   C  k_scan_drop   : bins above the threshold -> mask1 bit; the threshold bin's
//                      elements -> candidate list; everything below contributes
//                      to the grow histogram (same pass reads the dense grad)
//   D  k_resolve<0>  : per layer: a level-2 histogram (next 12 key bits, filled by C)
//                      narrows the candidates to a handful; those are ranked exactly
//                      on the 52-bit composite (low 20 key bits, inverted index) in
//                      shared memory -> exact cut incl. tie-break (a global radix
//                      select is the fallback for huge tie groups); completes the
//                      grow histogram; picks the grow threshold bin
//   E  k_scan_grow   : definite grows -> mask2 bit, weight/slot re-init at new
//                      connections; threshold bin -> block-private candidate lists
//   F  k_resolve<1>  : exact grow cut (a 52-bit threshold per layer)
//   G  k_publish_mask: every scan block applies the cut to its own candidate list
//                      (bit + re-init), then mask = mask1 | mask2 for its chunk
// Selection is by exact integer comparison of (key, index) composites, hence
// deterministic and independent of atomic ordering.
//
// HBM traffic (algorithmic floor 8.25 N bytes, SURVEY 8d): A reads 4N (+N/8),
// C reads 8N, E reads 4N (+bitmaps) => ~16.4 N with no noise tensor.  The three scans
// (A, C, E) are NOT HBM-bound: ~2 warp instructions per element at 0.4 IPC per
// scheduler, and a block's duration is its dependent chain of load -> classify trips,
// so the scan block is small (8192 elements: ~5 waves instead of 1.3 of 4x longer
// blocks; measured 0.36 -> 0.30 ms for the sequence).  Cutting the shared-memory
// histogram atomics 8x (a sampled floor under the grow threshold, validated in-kernel)
// was built and measured: 125 -> 112 us for C, paid back by the sampling -- not kept.
#include <algorithm>
#include <cstdlib>
#include <vector>

#include "common.cuh"

namespace rigl {

constexpr int kBins = 4096;
constexpr int kBinShift = 20;
constexpr uint32_t kKeyZero = 0x80000000u;  // ord_key(+0.0f)
constexpr int kScanThreads = 256;
constexpr int kGroup = 128;                 // elements per warp-iteration (float4 per lane)
constexpr int kChunk = 8192;                // default elements per scan block (plan->chunk; env RIGL_MASK_CHUNK)
constexpr int kResolveThreads = 1024;
constexpr int kRBins = 2048;
constexpr int kBatch = 2;                   // groups whose loads are issued together per trip

struct LayerState {     // 64 bytes, zeroed at the start of every run
  int32_t n_ones, n_prune, n_keep, n_cand_drop;
  int32_t n_cand_grow, drop_bucket, grow_bucket, n_ones_acc;
  uint32_t drop_need, grow_need, cand_cnt_drop, cand_cnt_grow;
  int32_t n_grow;          // connections to grow: n_prune, or 0 with RIGL_LAYER_DROP_ONLY
  uint32_t pad1;
  uint32_t grow_thresh_lo, grow_thresh_hi;   // exact grow cut (52-bit composite), applied by k_publish_mask
};

struct LayerDev {
  float* w;
  const float* g;
  uint32_t* mask;
  const float* noise;
  float* slot0;
  float* slot1;
  const float* grow;
  const float* sdrop;
  const float* grad;      // gradient for grad_scale / grad_sign init and the slot reset (null: score_grow is it)
  uint32_t flags;         // RIGL_LAYER_* bits
  uint32_t noise_key;     // per-layer key of the in-kernel drop-score noise
  uint32_t n;
  int32_t n_prune_override;
  uint64_t off_mask1;   // byte offsets into the workspace
  uint64_t off_hist_drop;
  uint64_t off_hist_grow;
  uint64_t off_hist2_drop;   // level-2 histograms (key bits 19..8 of the threshold bin's elements)
  uint64_t off_hist2_grow;
  uint64_t off_cand;
  uint64_t off_state;
  uint32_t first_task;  // this layer's blocks are tasks[first_task .. first_task + n_tasks)
  uint32_t n_tasks;
};

struct BlockTask {
  uint32_t layer;
  uint32_t start;
};

struct RunParams {
  float drop_fraction;
  int grow_mode;
  float grow_divisor;
  float acc_scale;
  int reinit_when_same;
  float noise_std;            // > 0: layers without a noise tensor draw N(0, noise_std) in-kernel
  uint32_t seed_lo, seed_hi;  // run key of that draw (seed offset + hash | global step)
  uint64_t off_task_cnt;      // workspace offset of the grow candidates per scan block: [n_blocks]
  uint32_t n_blocks;
  uint32_t chunk;             // elements per scan block (a multiple of 4096)
};

// Counter-based N(0,1) noise for the drop scores (generic_mask_update's `noise_std`, base.py:260-274, 523-538):
// element i of a layer takes one half of a Box-Muller pair from Philox2x32-10(counter = (i >> 1, seed_hi),
// key = layer_key ^ seed_lo).  No tensor is written or read: the two scans that need the noise recompute it.
// Every fp op is an explicit round-to-nearest intrinsic or a MUFU approximation, so the value of element i is the
// same in every kernel (and in rigl_mask_noise_fill, which materialises it for the tests / the oracle).
__device__ __forceinline__ void philox2x32_10(uint32_t c0, uint32_t c1, uint32_t key, uint32_t& o0, uint32_t& o1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi = __umulhi(0xD256D193u, c0), lo = 0xD256D193u * c0;
    c0 = hi ^ key ^ c1;
    c1 = lo;
    key += 0x9E3779B9u;
  }
  o0 = c0; o1 = c1;
}

__device__ __forceinline__ float2 normal_pair(uint32_t pair_idx, uint32_t layer_key, uint32_t seed_lo, uint32_t seed_hi) {
  uint32_t x0, x1;
  philox2x32_10(pair_idx, seed_hi, layer_key ^ seed_lo, x0, x1);
  const float u1 = __fmul_rn((float)((x0 >> 8) + 1u), 5.9604644775390625e-08f);      // (0, 1]
  const float u2 = __fmul_rn((float)(x1 >> 8), 5.9604644775390625e-08f);             // [0, 1)
  const float r = __fsqrt_rn(__fmul_rn(-2.0f, __logf(u1)));
  const float th = __fmul_rn(6.2831853071795864769f, u2);
  return make_float2(__fmul_rn(r, __cosf(th)), __fmul_rn(r, __sinf(th)));
}

// noise of elements e0 .. e0+3 (e0 a multiple of 4)
__device__ __forceinline__ float4 noise4(uint32_t e0, uint32_t layer_key, const RunParams& prm) {
  const float2 a = normal_pair(e0 >> 1, layer_key, prm.seed_lo, prm.seed_hi);
  const float2 b = normal_pair((e0 >> 1) + 1u, layer_key, prm.seed_lo, prm.seed_hi);
  return make_float4(__fmul_rn(a.x, prm.noise_std), __fmul_rn(a.y, prm.noise_std), __fmul_rn(b.x, prm.noise_std),
                     __fmul_rn(b.y, prm.noise_std));
}

__global__ void k_noise_fill(float* __restrict__ out, uint32_t n, uint32_t layer_key, RunParams prm) {
  const uint32_t e0 = (blockIdx.x * blockDim.x + threadIdx.x) * 4u;
  if (e0 >= n) return;
  const float4 v = noise4(e0, layer_key, prm);
  const float vs[4] = {v.x, v.y, v.z, v.w};
  for (int c = 0; c < 4 && e0 + c < n; ++c) out[e0 + c] = vs[c];
}

__device__ __forceinline__ float4 load4_guard(const float* __restrict__ p, uint32_t e0, uint32_t n) {
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (e0 + 3 < n) {
    v = __ldg(reinterpret_cast<const float4*>(p + e0));
  } else {
    if (e0 < n) v.x = __ldg(p + e0);
    if (e0 + 1 < n) v.y = __ldg(p + e0 + 1);
    if (e0 + 2 < n) v.z = __ldg(p + e0 + 2);
  }
  return v;
}

// grow ranking key: |score| for the RigL / Momentum callers (the score IS the dense gradient and the reference
// ranks abs(grad), base.py:529), the score verbatim for `_get_update_op(score_drop, score_grow, ...)`
__device__ __forceinline__ uint32_t grow_key(float g, bool is_signed) {
  return ord_key(is_signed ? g : fabsf(g));
}

__device__ __forceinline__ float drop_score(float w, uint32_t bit, float noise, bool has_noise,
                                            bool explicit_score) {
  if (explicit_score) return w;      // caller-supplied score_drop, used verbatim
  float s = bit ? fabsf(w) : 0.0f;
  if (has_noise) s = __fadd_rn(s, noise);
  return s;
}

// OR-combine 4-bit nibbles of 8 consecutive lanes into one 32-bit word
// (lane l owns elements 4l..4l+3 of a 128-element group).
__device__ __forceinline__ uint32_t combine_nibbles(uint32_t nib, int lane) {
  uint32_t v = nib << (4 * (lane & 7));
  v |= __shfl_xor_sync(0xffffffffu, v, 1);
  v |= __shfl_xor_sync(0xffffffffu, v, 2);
  v |= __shfl_xor_sync(0xffffffffu, v, 4);
  return v;
}

__device__ __forceinline__ void flush_hist(const uint32_t* sh, uint32_t* gh) {
  for (int b = threadIdx.x; b < kBins; b += blockDim.x) {
    uint32_t v = sh[b];
    if (v) atomicAdd(gh + b, v);
  }
}

// ----------------------------------------------------------------------------
// A: histogram of drop keys
// ----------------------------------------------------------------------------
template <bool kGenNoise>       // in-kernel noise is a separate instantiation: the plain path keeps its schedule
__global__ void __launch_bounds__(kScanThreads, 4)
k_hist_drop(const LayerDev* __restrict__ layers, const BlockTask* __restrict__ tasks, uint8_t* ws, RunParams prm) {
  __shared__ uint32_t hist[kBins];
  const BlockTask task = tasks[blockIdx.x];
  const LayerDev L = layers[task.layer];
  LayerState* st = reinterpret_cast<LayerState*>(ws + L.off_state);
  for (int b = threadIdx.x; b < kBins; b += kScanThreads) hist[b] = 0;
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool explicit_score = L.sdrop != nullptr;
  const bool gen_noise = kGenNoise && L.noise == nullptr && !explicit_score && prm.noise_std > 0.f;
  const bool has_noise = (L.noise != nullptr && !explicit_score) || gen_noise;
  const float* __restrict__ wsrc = explicit_score ? L.sdrop : L.w;
  const uint32_t n = L.n;
  const bool all_active = (L.flags & RIGL_LAYER_ALL_ACTIVE) != 0;     // rank every position (mask treated as ones)
  uint32_t zero_cnt = 0, ones = 0;
  constexpr int kWarps = kScanThreads / 32;
  const int kTrips = (int)prm.chunk / kGroup / kWarps;    // groups per warp
#pragma unroll 1
  for (int j0 = 0; j0 < kTrips; j0 += kBatch) {
    // issue the loads of 4 groups before touching any of them (memory-level parallelism)
    float4 wv[kBatch], nv[kBatch];
    uint32_t mw[kBatch], e0s[kBatch];
    bool act[kBatch];
#pragma unroll
    for (int u = 0; u < kBatch; ++u) {
      const uint32_t base = task.start + (uint32_t)(warp + kWarps * (j0 + u)) * kGroup;
      act[u] = base < n;                                  // warp-uniform
      e0s[u] = base + 4 * lane;
      nv[u] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (act[u]) {
        wv[u] = load4_guard(wsrc, e0s[u], n);
        if (gen_noise) nv[u] = noise4(e0s[u], L.noise_key, prm);
        else if (has_noise) nv[u] = load4_guard(L.noise, e0s[u], n);
        mw[u] = __ldg(L.mask + (base >> 5) + (lane >> 3));
      }
    }
#pragma unroll
    for (int u = 0; u < kBatch; ++u) {
      if (!act[u]) continue;
      if ((lane & 7) == 0) ones += __popc(mw[u]);
      const uint32_t nib = all_active ? 0xFu : (mw[u] >> (4 * (lane & 7))) & 0xFu;
      const float ws4[4] = {wv[u].x, wv[u].y, wv[u].z, wv[u].w};
      const float ns4[4] = {nv[u].x, nv[u].y, nv[u].z, nv[u].w};
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        if (e0s[u] + c < n) {
          const uint32_t key = ord_key(drop_score(ws4[c], (nib >> c) & 1u, ns4[c], has_noise, explicit_score));
          if (key == kKeyZero) ++zero_cnt;         // masked-out entries: avoid a 32-way smem hot spot
          else atomicAdd(&hist[key >> kBinShift], 1u);
        }
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    zero_cnt += __shfl_xor_sync(0xffffffffu, zero_cnt, o);
    ones += __shfl_xor_sync(0xffffffffu, ones, o);
  }
  if (lane == 0) {
    if (zero_cnt) atomicAdd(&hist[kKeyZero >> kBinShift], zero_cnt);
    if (ones) atomicAdd(&st->n_ones_acc, (int32_t)ones);        // popcount(mask) for free
  }
  __syncthreads();
  flush_hist(hist, reinterpret_cast<uint32_t*>(ws + L.off_hist_drop));
}

// ----------------------------------------------------------------------------
// Block-wide helpers for the per-layer kernels (1024 threads)
// ----------------------------------------------------------------------------
__device__ __forceinline__ uint32_t block_inclusive_scan(uint32_t v, uint32_t* warp_sums /*[32]*/) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    uint32_t t = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += t;
  }
  if (lane == 31) warp_sums[warp] = v;
  __syncthreads();
  if (warp == 0) {
    uint32_t s = warp_sums[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      uint32_t t = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += t;
    }
    warp_sums[lane] = s;
  }
  __syncthreads();
  if (warp > 0) v += warp_sums[warp - 1];
  __syncthreads();
  return v;
}

// Finds, scanning bins from the highest down, the bin where the running count
// reaches `need` (need >= 1, total >= need).  hist has NB bins in shared memory,
// NB = kResolveThreads * PER.  Result via shared out[3] = {bin, need_in_bin, count_in_bin}.
template <int NB>
__device__ __forceinline__ void find_bin_desc(const uint32_t* hist, uint32_t need, uint32_t* warp_sums,
                                              uint32_t* out) {
  constexpr int PER = NB / kResolveThreads;
  const int t = threadIdx.x;
  uint32_t local[PER];
  uint32_t s = 0;
#pragma unroll
  for (int j = 0; j < PER; ++j) {
    local[j] = hist[NB - 1 - (t * PER + j)];
    s += local[j];
  }
  const uint32_t incl = block_inclusive_scan(s, warp_sums);
  uint32_t run = incl - s;
  if (run < need && need <= incl) {
#pragma unroll
    for (int j = 0; j < PER; ++j) {
      if (run < need && need <= run + local[j]) {
        out[0] = NB - 1 - (t * PER + j);
        out[1] = need - run;
        out[2] = local[j];
      }
      run += local[j];
    }
  }
  __syncthreads();
}

// ----------------------------------------------------------------------------
// B: per-layer counts and drop threshold bin
// ----------------------------------------------------------------------------
__global__ void __launch_bounds__(kResolveThreads)
k_pick_drop(const LayerDev* __restrict__ layers, uint8_t* ws, RunParams prm) {
  __shared__ uint32_t hist[kBins];
  __shared__ uint32_t warp_sums[32];
  __shared__ uint32_t out[3];
  __shared__ int32_t s_counts[2];
  const LayerDev L = layers[blockIdx.x];
  LayerState* st = reinterpret_cast<LayerState*>(ws + L.off_state);
  const uint32_t* gh = reinterpret_cast<const uint32_t*>(ws + L.off_hist_drop);
  for (int b = threadIdx.x; b < kBins; b += kResolveThreads) hist[b] = __ldcg(gh + b);
  __syncthreads();
  if (threadIdx.x == kResolveThreads - 1) {
    const int32_t n_ones = (L.flags & RIGL_LAYER_ALL_ACTIVE) ? (int32_t)L.n
                                                             : st->n_ones_acc;   // accumulated by k_hist_drop
    int32_t n_prune = L.n_prune_override >= 0
                          ? L.n_prune_override
                          : (int32_t)__fmul_rn((float)n_ones, prm.drop_fraction);  // base.py:287-289
    if (n_prune > n_ones) n_prune = n_ones;
    if (n_prune < 0) n_prune = 0;
    s_counts[0] = n_ones - n_prune;
    s_counts[1] = n_prune;
    st->n_ones = n_ones;
    st->n_prune = n_prune;
    st->n_keep = n_ones - n_prune;
    st->n_grow = (L.flags & RIGL_LAYER_DROP_ONLY) ? 0 : n_prune;
  }
  if (threadIdx.x == 0) { out[0] = kBins; out[1] = 0; out[2] = 0; }
  __syncthreads();
  const uint32_t n_keep = (uint32_t)s_counts[0];
  if (n_keep > 0) find_bin_desc<kBins>(hist, n_keep, warp_sums, out);
  if (threadIdx.x == 0) {
    st->drop_bucket = (int32_t)out[0];   // kBins => nothing kept
    st->drop_need = out[1];
    st->n_cand_drop = (int32_t)out[2];
  }
}

// Appends one warp's candidates of a 128-element group to a candidate list: lane holds up to four (bit c of nibc set
// <=> element e0 + c, key keys[c]).  One warp scan + ONE counter atomic per group (instead of a ballot, an atomic and a
// shuffle per element column); the order inside the list is irrelevant to the selection.
__device__ __forceinline__ void append_cands(uint32_t nibc, const uint32_t (&keys)[4], uint32_t e0, int lane,
                                             uint2* __restrict__ cand, uint32_t* counter, uint32_t* __restrict__ hist2) {
  if (!__any_sync(0xffffffffu, nibc != 0u)) return;
  const uint32_t mine = __popc(nibc);
  uint32_t incl = mine;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  uint32_t base = 0;
  if (lane == 31) base = atomicAdd(counter, incl);     // global (one list per layer) or shared (block-private list)
  base = __shfl_sync(0xffffffffu, base, 31);
  uint32_t pos = base + incl - mine;
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    if ((nibc >> c) & 1u) {
      cand[pos++] = make_uint2(keys[c], e0 + c);
      atomicAdd(&hist2[(keys[c] >> 8) & 0xFFFu], 1u);
    }
  }
}

// ----------------------------------------------------------------------------
// C: classify against the drop threshold bin, build mask1, grow histogram
// ----------------------------------------------------------------------------
// (drop candidates are rare -- the threshold bin of the ~20 % active weights -- and go to ONE list per layer)
template <bool kGenNoise>
__global__ void __launch_bounds__(kScanThreads, 4)
k_scan_drop(const LayerDev* __restrict__ layers, const BlockTask* __restrict__ tasks, uint8_t* ws, RunParams prm) {
  __shared__ uint32_t hist[kBins];
  const BlockTask task = tasks[blockIdx.x];
  const LayerDev L = layers[task.layer];
  LayerState* st = reinterpret_cast<LayerState*>(ws + L.off_state);
  uint32_t* mask1 = reinterpret_cast<uint32_t*>(ws + L.off_mask1);
  uint32_t* hist2 = reinterpret_cast<uint32_t*>(ws + L.off_hist2_drop);
  uint2* cand = reinterpret_cast<uint2*>(ws + L.off_cand);
  for (int b = threadIdx.x; b < kBins; b += kScanThreads) hist[b] = 0;
  __syncthreads();
  const uint32_t bucket = (uint32_t)st->drop_bucket;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool explicit_score = L.sdrop != nullptr;
  const bool gen_noise = kGenNoise && L.noise == nullptr && !explicit_score && prm.noise_std > 0.f;
  const bool has_noise = (L.noise != nullptr && !explicit_score) || gen_noise;
  const float* __restrict__ wsrc = explicit_score ? L.sdrop : L.w;
  const uint32_t n = L.n;
  const bool grow_signed = (L.flags & RIGL_LAYER_GROW_SCORE_SIGNED) != 0;
  const bool all_active = (L.flags & RIGL_LAYER_ALL_ACTIVE) != 0;
  uint32_t zero_cnt = 0;
  constexpr int kWarps = kScanThreads / 32;
  const int kTrips = (int)prm.chunk / kGroup / kWarps;
#pragma unroll 1
  for (int j0 = 0; j0 < kTrips; j0 += kBatch) {
    float4 wv[kBatch], gv[kBatch], nv[kBatch];
    uint32_t mw[kBatch], bases[kBatch];
    bool act[kBatch];
#pragma unroll
    for (int u = 0; u < kBatch; ++u) {
      bases[u] = task.start + (uint32_t)(warp + kWarps * (j0 + u)) * kGroup;
      act[u] = bases[u] < n;
      nv[u] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (act[u]) {
        const uint32_t e0 = bases[u] + 4 * lane;
        wv[u] = load4_guard(wsrc, e0, n);
        gv[u] = load4_guard(L.g, e0, n);
        if (gen_noise) nv[u] = noise4(e0, L.noise_key, prm);
        else if (has_noise) nv[u] = load4_guard(L.noise, e0, n);
        mw[u] = __ldg(L.mask + (bases[u] >> 5) + (lane >> 3));
      }
    }
#pragma unroll
    for (int u = 0; u < kBatch; ++u) {
      if (!act[u]) continue;
      const uint32_t e0 = bases[u] + 4 * lane;
      const uint32_t nib = all_active ? 0xFu : (mw[u] >> (4 * (lane & 7))) & 0xFu;
      const float ws4[4] = {wv[u].x, wv[u].y, wv[u].z, wv[u].w};
      const float gs4[4] = {gv[u].x, gv[u].y, gv[u].z, gv[u].w};
      const float ns4[4] = {nv[u].x, nv[u].y, nv[u].z, nv[u].w};
      uint32_t nib1 = 0, nibc = 0;
      uint32_t keys[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const bool valid = e0 + c < n;
        uint32_t key = 0, bin = 0;
        if (valid) {
          key = ord_key(drop_score(ws4[c], (nib >> c) & 1u, ns4[c], has_noise, explicit_score));
          bin = key >> kBinShift;
        }
        keys[c] = key;
        const bool is_cand = valid && bin == bucket;
        const bool kept = valid && bin > bucket;
        if (kept) nib1 |= 1u << c;
        if (is_cand) nibc |= 1u << c;
        if (valid && !kept && !is_cand) {          // definitely dropped / inactive: a grow contender
          const uint32_t gkey = grow_key(gs4[c], grow_signed);
          if (gkey == kKeyZero) ++zero_cnt;
          else atomicAdd(&hist[gkey >> kBinShift], 1u);
        }
      }
      append_cands(nibc, keys, e0, lane, cand, &st->cand_cnt_drop, hist2);
      const uint32_t word = combine_nibbles(nib1, lane);
      if ((lane & 7) == 0) mask1[(bases[u] >> 5) + (lane >> 3)] = word;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) zero_cnt += __shfl_xor_sync(0xffffffffu, zero_cnt, o);
  if (lane == 0 && zero_cnt) atomicAdd(&hist[kKeyZero >> kBinShift], zero_cnt);
  __syncthreads();
  flush_hist(hist, reinterpret_cast<uint32_t*>(ws + L.off_hist_grow));
}

// ----------------------------------------------------------------------------
// Apply helpers: what happens at a newly grown connection
// ----------------------------------------------------------------------------
__device__ __forceinline__ void apply_new_connection(const LayerDev& L, const RunParams& prm, uint32_t e,
                                                     float g) {
  if (L.grad) g = __ldg(L.grad + e);
  float v = 0.0f;
  switch (prm.grow_mode) {
    case RIGL_GROW_TENSOR: v = __ldg(L.grow + e); break;
    case RIGL_GROW_GRAD_SCALE: v = __fdiv_rn(g, prm.grow_divisor); break;
    case RIGL_GROW_GRAD_SIGN:
      v = __fdiv_rn(g > 0.f ? 1.0f : (g < 0.f ? -1.0f : g), prm.grow_divisor);
      break;
    default: break;
  }
  L.w[e] = v;
  const float r = __fmul_rn(g, prm.acc_scale);
  if (L.slot0) L.slot0[e] = r;
  if (L.slot1) L.slot1[e] = r;
}

// ----------------------------------------------------------------------------
// D / F: exact cut inside the threshold bin (per layer, one block)
// ----------------------------------------------------------------------------
__device__ __forceinline__ uint64_t composite(uint2 c) {
  return ((uint64_t)(c.x & 0xFFFFFu) << 32) | (uint64_t)(0xFFFFFFFFu - c.y);
}

constexpr int kSubCap = 1024;      // sub-candidates ranked exactly in shared memory

// Visits every candidate of a layer with the whole block.  One list per layer (cnt entries: drop), or one list per
// scan block (blk_cnt[b] entries at cand + b * chunk: grow) -- a warp per list, lanes striding over it.
template <bool kLists, typename F>
__device__ __forceinline__ void for_each_cand(const uint2* __restrict__ cand, uint32_t cnt,
                                              const uint32_t* __restrict__ blk_cnt, uint32_t n_lists, uint32_t chunk,
                                              F&& f) {
  if (!kLists) {
    for (uint32_t i = threadIdx.x; i < cnt; i += kResolveThreads) f(cand[i]);
  } else {
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (uint32_t b = warp; b < n_lists; b += kResolveThreads / 32) {
      const uint32_t c = __ldcg(blk_cnt + b);
      const uint2* lst = cand + (size_t)b * chunk;
      for (uint32_t i = lane; i < c; i += 32) f(lst[i]);
    }
  }
}

template <bool kGrow>
__global__ void __launch_bounds__(kResolveThreads)
k_resolve(const LayerDev* __restrict__ layers, uint8_t* ws, RunParams prm) {
  __shared__ uint32_t h2[kBins];                 // level-2 histogram; reused as the fallback radix histogram
  __shared__ uint32_t ghist[kGrow ? 1 : kBins];
  __shared__ uint2 sub[kSubCap];
  __shared__ uint32_t warp_sums[32];
  __shared__ uint32_t out[3];
  __shared__ uint32_t sub_cnt;
  __shared__ unsigned long long s_thresh;
  const LayerDev L = layers[blockIdx.x];
  LayerState* st = reinterpret_cast<LayerState*>(ws + L.off_state);
  uint32_t* mask1 = reinterpret_cast<uint32_t*>(ws + L.off_mask1);
  const uint2* cand = reinterpret_cast<const uint2*>(ws + L.off_cand);
  const uint32_t cnt = kGrow ? st->cand_cnt_grow : st->cand_cnt_drop;
  uint32_t need = kGrow ? st->grow_need : st->drop_need;
  const int tid = threadIdx.x;
  const uint32_t* blk_cnt = reinterpret_cast<const uint32_t*>(ws + prm.off_task_cnt) + L.first_task;   // (grow)

  {
    const uint32_t* g2 = reinterpret_cast<const uint32_t*>(ws + (kGrow ? L.off_hist2_grow : L.off_hist2_drop));
    for (int b = tid; b < kBins; b += kResolveThreads) h2[b] = __ldcg(g2 + b);
  }
  if (!kGrow) {
    const uint32_t* gh = reinterpret_cast<const uint32_t*>(ws + L.off_hist_grow);
    for (int b = tid; b < kBins; b += kResolveThreads) ghist[b] = __ldcg(gh + b);
  }
  if (tid == 0) { sub_cnt = 0; s_thresh = 0ull; }
  __syncthreads();

  // --- the cut: selected <=> composite >= thresh ---
  uint64_t thresh = 0;
  if (need == 0) thresh = ~0ull;       // nothing (composites use 52 bits)
  if (need > 0 && need < cnt) {
    find_bin_desc<kBins>(h2, need, warp_sums, out);           // level 2: key bits 19..8
    const uint32_t b2 = out[0];
    need = out[1];
    const uint32_t in_bin = out[2];
    __syncthreads();
    thresh = (uint64_t)b2 << 40;
    if (in_bin != need) {
      // gather the elements of the level-2 threshold bin
      for_each_cand<kGrow>(cand, cnt, blk_cnt, L.n_tasks, prm.chunk, [&](const uint2 c) {
        if (((c.x >> 8) & 0xFFFu) == b2) {
          const uint32_t pos = atomicAdd(&sub_cnt, 1u);
          if (pos < (uint32_t)kSubCap) sub[pos] = c;
        }
      });
      __syncthreads();
      const uint32_t ns = sub_cnt;
      if (ns <= (uint32_t)kSubCap) {
        // exact rank inside shared memory: the need-th largest composite is the threshold
        if ((uint32_t)tid < ns) {
          const uint64_t mine = composite(sub[tid]);
          uint32_t rank = 0;
          for (uint32_t j = 0; j < ns; ++j) rank += composite(sub[j]) > mine;
          if (rank == need - 1) s_thresh = mine;
        }
        __syncthreads();
        thresh = s_thresh;
      } else {
        // huge tie group: radix select over the whole candidate list on the remaining 40 bits
        const int shifts[4] = {29, 18, 7, 0};
        const int widths[4] = {11, 11, 11, 7};
        uint64_t prefix = b2;
#pragma unroll 1
        for (int p = 0; p < 4; ++p) {
          const int sh = shifts[p], wd = widths[p];
          for (int b = tid; b < kRBins; b += kResolveThreads) h2[b] = 0;
          __syncthreads();
          for_each_cand<kGrow>(cand, cnt, blk_cnt, L.n_tasks, prm.chunk, [&](const uint2 cc) {
            const uint64_t c = composite(cc);
            if ((c >> (sh + wd)) == prefix) atomicAdd(&h2[(uint32_t)(c >> sh) & ((1u << wd) - 1u)], 1u);
          });
          __syncthreads();
          find_bin_desc<kRBins>(h2, need, warp_sums, out);
          prefix = (prefix << wd) | out[0];
          need = out[1];
          const uint32_t inb = out[2];
          __syncthreads();
          thresh = prefix << sh;
          if (inb == need) break;       // every composite with this prefix is selected
        }
      }
    }
  }
  __syncthreads();

  if constexpr (kGrow) {
    // the grow cut is applied by k_publish_mask, every scan block to its own list (one block per layer walking
    // ~40 k candidates and copying a 2.4 M-bit bitmap was most of this kernel's time)
    if (tid == 0) { st->grow_thresh_lo = (uint32_t)thresh; st->grow_thresh_hi = (uint32_t)(thresh >> 32); }
  } else {
    // --- act on the drop candidates: kept -> mask1 bit; dropped -> a grow contender ---
    for_each_cand<false>(cand, cnt, blk_cnt, L.n_tasks, prm.chunk, [&](const uint2 c) {
      const uint32_t e = c.y;
      if (composite(c) >= thresh) {
        atomicOr(mask1 + (e >> 5), 1u << (e & 31));
      } else {
        const uint32_t gkey = grow_key(__ldg(L.g + e), (L.flags & RIGL_LAYER_GROW_SCORE_SIGNED) != 0);
        atomicAdd(&ghist[gkey >> kBinShift], 1u);
      }
    });
    __syncthreads();
    // grow threshold bin: top-n_prune among positions with mask1 == 0
    if (tid == 0) { out[0] = kBins; out[1] = 0; out[2] = 0; }
    __syncthreads();
    const uint32_t n_grow = (uint32_t)st->n_grow;
    if (n_grow > 0) find_bin_desc<kBins>(ghist, n_grow, warp_sums, out);
    if (tid == 0) {
      st->grow_bucket = (int32_t)out[0];
      st->grow_need = out[1];
      st->n_cand_grow = (int32_t)out[2];
    }
  }
}

// G: applies the exact grow cut to this block's own candidate list (bit into mask1 + re-initialisation; every
// candidate of the list lies in this block's chunk of the bitmap, so the OR-ed bits are complete before the copy),
// then mask <- mask1 (| mask2, already OR-ed in by k_scan_grow) for the chunk.  All layers, full grid.
__global__ void __launch_bounds__(kScanThreads)
k_publish_mask(const LayerDev* __restrict__ layers, const BlockTask* __restrict__ tasks, uint8_t* ws,
               RunParams prm) {
  const BlockTask task = tasks[blockIdx.x];
  const LayerDev L = layers[task.layer];
  uint32_t* mask1 = reinterpret_cast<uint32_t*>(ws + L.off_mask1);
  {
    const LayerState* st = reinterpret_cast<const LayerState*>(ws + L.off_state);
    const uint32_t c = reinterpret_cast<const uint32_t*>(ws + prm.off_task_cnt)[blockIdx.x];
    if (c > 0 && st->n_grow > 0) {
      const uint64_t thresh = ((uint64_t)st->grow_thresh_hi << 32) | (uint64_t)st->grow_thresh_lo;
      const uint2* lst = reinterpret_cast<const uint2*>(ws + L.off_cand) + task.start;
      for (uint32_t i = threadIdx.x; i < c; i += kScanThreads) {
        const uint2 cd = lst[i];
        if (composite(cd) >= thresh) {
          const uint32_t e = cd.y;
          atomicOr(mask1 + (e >> 5), 1u << (e & 31));
          const bool was_on = (L.mask[e >> 5] >> (e & 31)) & 1u;     // the old mask (overwritten below: no __ldg)
          if (!was_on || prm.reinit_when_same) apply_new_connection(L, prm, e, __ldg(L.g + e));
        }
      }
    }
    __syncthreads();
  }
  const uint32_t words = (L.n + 31) >> 5;
  const uint32_t w0 = task.start >> 5;
  for (uint32_t i = w0 + threadIdx.x; i < min(words, w0 + (prm.chunk >> 5)); i += kScanThreads)
    L.mask[i] = __ldcg(mask1 + i);
}

// ----------------------------------------------------------------------------
// E: classify against the grow threshold bin
// ----------------------------------------------------------------------------
// Grow candidates (a few % of ALL positions) go to a block-private list: cand + task.start, at most `chunk` entries,
// the position from a shared-memory counter, the per-block count to task_cnt[] -- one list per layer would hang every
// group of every warp of the layer on the round trip of one global atomic (measured: 99 vs 71 us for this kernel).
__global__ void __launch_bounds__(kScanThreads, 4)
k_scan_grow(const LayerDev* __restrict__ layers, const BlockTask* __restrict__ tasks, uint8_t* ws,
            RunParams prm) {
  __shared__ uint32_t s_cand;
  constexpr int kGrowBatch = 4;                       // loads of 4 groups in flight (this scan holds few registers)
  const BlockTask task = tasks[blockIdx.x];
  const LayerDev L = layers[task.layer];
  LayerState* st = reinterpret_cast<LayerState*>(ws + L.off_state);
  uint32_t* mask1 = reinterpret_cast<uint32_t*>(ws + L.off_mask1);
  uint32_t* hist2 = reinterpret_cast<uint32_t*>(ws + L.off_hist2_grow);
  uint2* cand = reinterpret_cast<uint2*>(ws + L.off_cand) + task.start;
  if (st->n_grow == 0) return;                        // nothing grows; mask1 is final (block-uniform exit)
  if (threadIdx.x == 0) s_cand = 0;
  __syncthreads();
  const uint32_t bucket = (uint32_t)st->grow_bucket;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t n = L.n;
  const bool grow_signed = (L.flags & RIGL_LAYER_GROW_SCORE_SIGNED) != 0;
  constexpr int kWarps = kScanThreads / 32;
  const int kTrips = (int)prm.chunk / kGroup / kWarps;
#pragma unroll 1
  for (int j0 = 0; j0 < kTrips; j0 += kGrowBatch) {
    float4 gv[kGrowBatch];
    uint32_t m1w[kGrowBatch], oldw[kGrowBatch], bases[kGrowBatch];
    bool act[kGrowBatch];
#pragma unroll
    for (int u = 0; u < kGrowBatch; ++u) {
      bases[u] = task.start + (uint32_t)(warp + kWarps * (j0 + u)) * kGroup;
      act[u] = bases[u] < n;
      if (act[u]) {
        gv[u] = load4_guard(L.g, bases[u] + 4 * lane, n);
        const uint32_t widx = (bases[u] >> 5) + (lane >> 3);
        m1w[u] = __ldcg(mask1 + widx);
        oldw[u] = __ldg(L.mask + widx);
      }
    }
#pragma unroll
    for (int u = 0; u < kGrowBatch; ++u) {
      if (!act[u]) continue;
      const uint32_t e0 = bases[u] + 4 * lane;
      const uint32_t widx = (bases[u] >> 5) + (lane >> 3);
      const uint32_t nib_m1 = (m1w[u] >> (4 * (lane & 7))) & 0xFu;
      const uint32_t nib_old = (oldw[u] >> (4 * (lane & 7))) & 0xFu;
      const float gs4[4] = {gv[u].x, gv[u].y, gv[u].z, gv[u].w};
      uint32_t nib2 = 0, nibc = 0;
      uint32_t keys[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const bool contender = (e0 + c < n) && !((nib_m1 >> c) & 1u);
        uint32_t key = 0, bin = 0;
        if (contender) {
          key = grow_key(gs4[c], grow_signed);
          bin = key >> kBinShift;
        }
        keys[c] = key;
        if (contender && bin == bucket) nibc |= 1u << c;
        if (contender && bin > bucket) nib2 |= 1u << c;
      }
      // re-initialise the definitely grown connections: each lane walks its own set bits (usually 0 or 1 of 4), so the
      // warp runs the body ~1.5 times per group instead of once per element column
      uint32_t todo = prm.reinit_when_same ? nib2 : (nib2 & ~nib_old);
      while (todo) {
        const int c = __ffs(todo) - 1;
        todo &= todo - 1u;
        const float gc = c == 0 ? gv[u].x : (c == 1 ? gv[u].y : (c == 2 ? gv[u].z : gv[u].w));
        apply_new_connection(L, prm, e0 + c, gc);
      }
      append_cands(nibc, keys, e0, lane, cand, &s_cand, hist2);
      const uint32_t word2 = combine_nibbles(nib2, lane);
      if ((lane & 7) == 0 && word2) mask1[widx] = m1w[u] | word2;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const uint32_t c = s_cand;
    reinterpret_cast<uint32_t*>(ws + prm.off_task_cnt)[blockIdx.x] = c;
    if (c) atomicAdd(&st->cand_cnt_grow, c);
  }
}

// ----------------------------------------------------------------------------
// Gradual magnitude pruning (rigl_mask_prune_run): A-D with DROP_ONLY | ALL_ACTIVE and n_keep = k select the top k
// of |w|; these two kernels turn that cut into contrib's threshold and mask = |w| >= threshold (ties kept).
// ----------------------------------------------------------------------------
__device__ __forceinline__ float key_to_float(uint32_t key) {
  return __uint_as_float((key & 0x80000000u) ? (key ^ 0x80000000u) : ~key);
}

// Writes n_prune_override = n - k of up to kPruneCountBatch layers into the device layer table, from the kernel
// arguments (8 KB of parameters: CUDA 12.1+ on sm_70+ allows up to 32 KB).
constexpr int kPruneCountBatch = 2048;
struct PruneCounts {
  int32_t n_prune[kPruneCountBatch];
};

__global__ void k_prune_set_counts(LayerDev* __restrict__ layers, int first, int count, const PruneCounts counts) {
  for (int i = threadIdx.x; i < count; i += blockDim.x) layers[first + i].n_prune_override = counts.n_prune[i];
}

// H: per layer (one block): cur = the k-th largest |w| = the smallest key D kept.  Every kept position outside the
// drop threshold bin lies above it, and k >= 1 keeps at least one candidate of that bin, so the minimum over the
// kept candidates is the cut.  thr = cur * (1 - decay) + old * decay, each product and the sum rounded (no FMA).
__global__ void __launch_bounds__(kScanThreads)
k_prune_threshold(const LayerDev* __restrict__ layers, const uint8_t* __restrict__ ws, const float* old_thr,
                  float* new_thr, float decay) {      // (old_thr may alias new_thr)
  __shared__ uint32_t s_min;
  const LayerDev L = layers[blockIdx.x];
  const LayerState* st = reinterpret_cast<const LayerState*>(ws + L.off_state);
  const uint32_t* mask1 = reinterpret_cast<const uint32_t*>(ws + L.off_mask1);
  const uint2* cand = reinterpret_cast<const uint2*>(ws + L.off_cand);
  if (threadIdx.x == 0) s_min = 0xFFFFFFFFu;
  __syncthreads();
  const uint32_t cnt = st->cand_cnt_drop;
  uint32_t m = 0xFFFFFFFFu;
  for (uint32_t i = threadIdx.x; i < cnt; i += kScanThreads) {
    const uint2 c = cand[i];
    if ((__ldcg(mask1 + (c.y >> 5)) >> (c.y & 31)) & 1u) m = min(m, c.x);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = min(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMin(&s_min, m);
  __syncthreads();
  if (threadIdx.x == 0) {
    const float cur = key_to_float(s_min);
    new_thr[blockIdx.x] = __fadd_rn(__fmul_rn(cur, __fsub_rn(1.0f, decay)), __fmul_rn(old_thr[blockIdx.x], decay));
  }
}

// P: every scan block rewrites its chunk of the layer's bitmap as |w| >= thr.  All layers, full grid.
__global__ void __launch_bounds__(kScanThreads)
k_prune_publish(const LayerDev* __restrict__ layers, const BlockTask* __restrict__ tasks, const float* __restrict__ thr,
                RunParams prm) {
  const BlockTask task = tasks[blockIdx.x];
  const LayerDev L = layers[task.layer];
  const float t = thr[task.layer];
  const uint32_t n = L.n, words = (n + 31) >> 5;
  const uint32_t end = min(n, task.start + prm.chunk);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int kWarps = kScanThreads / 32;
#pragma unroll 4
  for (uint32_t base = task.start + (uint32_t)warp * kGroup; base < end; base += kWarps * kGroup) {
    const uint32_t e0 = base + 4 * lane;
    const float4 v = load4_guard(L.w, e0, n);
    const float ws4[4] = {v.x, v.y, v.z, v.w};
    uint32_t nib = 0;
#pragma unroll
    for (int c = 0; c < 4; ++c)
      if (e0 + c < n && fabsf(ws4[c]) >= t) nib |= 1u << c;
    const uint32_t word = combine_nibbles(nib, lane);
    const uint32_t widx = (base >> 5) + (lane >> 3);
    if ((lane & 7) == 0 && widx < words) L.mask[widx] = word;
  }
}

// ----------------------------------------------------------------------------
// Host side: plan
// ----------------------------------------------------------------------------
}  // namespace rigl

struct rigl_mask_plan {
  int n_layers = 0;
  int n_blocks = 0;
  rigl::LayerDev* d_layers = nullptr;
  rigl::BlockTask* d_tasks = nullptr;
  size_t ws_bytes = 0;
  size_t zero_bytes = 0;   // leading region memset to 0 each run (states + histograms + per-block counts)
  size_t state_off = 0;
  size_t task_cnt_off = 0; // [n_blocks] grow candidates per scan block
  int chunk = rigl::kChunk; // elements per scan block
  std::vector<rigl::LayerDev> h_layers;   // host copy of d_layers (rigl_mask_prune_run validates against it)
};

using namespace rigl;

static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

extern "C" int64_t rigl_mask_words(int64_t n) { return n <= 0 ? 0 : ((n + 127) / 128) * 4; }

extern "C" int rigl_mask_plan_create(const rigl_layer_desc* layers, int n_layers, rigl_mask_plan** out) {
  RIGL_REQUIRE(layers && out && n_layers > 0, "rigl_mask_plan_create: bad arguments");
  int64_t chunk = kChunk;
  if (const char* e = getenv("RIGL_MASK_CHUNK")) chunk = atoll(e);
  RIGL_REQUIRE(chunk >= 4096 && chunk <= (1 << 20) && chunk % 4096 == 0, "RIGL_MASK_CHUNK must be a multiple of 4096");
  std::vector<LayerDev> host(n_layers);
  std::vector<BlockTask> tasks;
  size_t off = 0;
  const size_t state_off = off;
  off += align_up(sizeof(LayerState) * (size_t)n_layers, 256);
  const size_t hist_drop_off = off;
  off += (size_t)n_layers * kBins * 4;
  const size_t hist_grow_off = off;
  off += (size_t)n_layers * kBins * 4;
  const size_t hist2_drop_off = off;
  off += (size_t)n_layers * kBins * 4;
  const size_t hist2_grow_off = off;
  off += (size_t)n_layers * kBins * 4;
  size_t total_tasks = 0;
  for (int l = 0; l < n_layers; ++l) {
    RIGL_REQUIRE(layers[l].n >= 1 && layers[l].n < (1ll << 31), "layer %d: n=%lld out of range", l, (long long)layers[l].n);
    total_tasks += (size_t)((layers[l].n + chunk - 1) / chunk);
  }
  const size_t task_cnt_off = off;
  off += align_up(total_tasks * sizeof(uint32_t), 256);
  const size_t zero_bytes = off;
  for (int l = 0; l < n_layers; ++l) {
    const rigl_layer_desc& d = layers[l];
    RIGL_REQUIRE(d.weights && d.score_grow && d.mask_bits, "layer %d: null tensor", l);
    RIGL_REQUIRE(aligned16(d.weights) && aligned16(d.score_grow) && aligned16(d.mask_bits) &&
                     aligned16(d.noise) && aligned16(d.score_drop) && aligned16(d.grad),
                 "layer %d: weights/score_grow/mask_bits/noise/score_drop must be 16-byte aligned", l);
    LayerDev& L = host[l];
    L.w = d.weights; L.g = d.score_grow; L.mask = d.mask_bits; L.noise = d.noise;
    L.slot0 = d.slots[0]; L.slot1 = d.slots[1]; L.grow = d.grow_values; L.sdrop = d.score_drop;
    L.grad = d.grad; L.flags = (uint32_t)d.flags; L.noise_key = d.noise_key;
    L.n = (uint32_t)d.n; L.n_prune_override = d.n_prune_override;
    L.off_state = state_off + sizeof(LayerState) * (size_t)l;
    L.off_hist_drop = hist_drop_off + (size_t)l * kBins * 4;
    L.off_hist_grow = hist_grow_off + (size_t)l * kBins * 4;
    L.off_hist2_drop = hist2_drop_off + (size_t)l * kBins * 4;
    L.off_hist2_grow = hist2_grow_off + (size_t)l * kBins * 4;
    L.off_mask1 = off;
    off += align_up((size_t)rigl_mask_words(d.n) * 4, 256);
    L.first_task = (uint32_t)tasks.size();
    for (int64_t s = 0; s < d.n; s += chunk) tasks.push_back({(uint32_t)l, (uint32_t)s});
    L.n_tasks = (uint32_t)tasks.size() - L.first_task;
  }
  for (int l = 0; l < n_layers; ++l) {
    host[l].off_cand = off;
    off += align_up((size_t)layers[l].n * sizeof(uint2), 256);
  }
  rigl_mask_plan* p = new rigl_mask_plan();
  p->n_layers = n_layers;
  p->n_blocks = (int)tasks.size();
  p->ws_bytes = off;
  p->zero_bytes = zero_bytes;
  p->state_off = state_off;
  p->task_cnt_off = task_cnt_off;
  p->chunk = (int)chunk;
  p->h_layers = host;
  cudaError_t e = cudaMalloc(&p->d_layers, sizeof(LayerDev) * n_layers);
  if (e == cudaSuccess) e = cudaMalloc(&p->d_tasks, sizeof(BlockTask) * tasks.size());
  if (e == cudaSuccess) e = cudaMemcpy(p->d_layers, host.data(), sizeof(LayerDev) * n_layers, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(p->d_tasks, tasks.data(), sizeof(BlockTask) * tasks.size(), cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    cudaFree(p->d_layers); cudaFree(p->d_tasks); delete p;
    return cuda_fail(e, "rigl_mask_plan_create");
  }
  *out = p;
  return RIGL_OK;
}

extern "C" int rigl_mask_plan_destroy(rigl_mask_plan* plan) {
  if (!plan) return RIGL_OK;
  cudaFree(plan->d_layers);
  cudaFree(plan->d_tasks);
  delete plan;
  return RIGL_OK;
}

extern "C" size_t rigl_mask_plan_workspace_bytes(const rigl_mask_plan* plan) {
  return plan ? plan->ws_bytes : 0;
}

static int check_workspace(const rigl_mask_plan* plan, const void* workspace, size_t workspace_bytes) {
  RIGL_REQUIRE(plan && workspace, "rigl_mask_update_run: null plan/workspace");
  if (workspace_bytes < plan->ws_bytes) {
    set_error("rigl_mask_update_run: workspace %zu < required %zu", workspace_bytes, plan->ws_bytes);
    return RIGL_ERR_WORKSPACE;
  }
  RIGL_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "workspace must be 256B aligned");
  return RIGL_OK;
}

// zero the workspace's state region, then A-D: the drop cut of every layer (mask1 = the kept set)
static int launch_drop_select(rigl_mask_plan* plan, RunParams& prm, uint8_t* ws, cudaStream_t stream) {
  RIGL_CUDA(cudaMemsetAsync(ws, 0, plan->zero_bytes, stream));
  prm.off_task_cnt = plan->task_cnt_off;
  prm.n_blocks = (uint32_t)plan->n_blocks;
  prm.chunk = (uint32_t)plan->chunk;
  const bool gen = prm.noise_std > 0.f;
  if (gen) k_hist_drop<true><<<plan->n_blocks, kScanThreads, 0, stream>>>(plan->d_layers, plan->d_tasks, ws, prm);
  else k_hist_drop<false><<<plan->n_blocks, kScanThreads, 0, stream>>>(plan->d_layers, plan->d_tasks, ws, prm);
  RIGL_LAUNCH_CHECK("k_hist_drop");
  k_pick_drop<<<plan->n_layers, kResolveThreads, 0, stream>>>(plan->d_layers, ws, prm);
  RIGL_LAUNCH_CHECK("k_pick_drop");
  if (gen) k_scan_drop<true><<<plan->n_blocks, kScanThreads, 0, stream>>>(plan->d_layers, plan->d_tasks, ws, prm);
  else k_scan_drop<false><<<plan->n_blocks, kScanThreads, 0, stream>>>(plan->d_layers, plan->d_tasks, ws, prm);
  RIGL_LAUNCH_CHECK("k_scan_drop");
  k_resolve<false><<<plan->n_layers, kResolveThreads, 0, stream>>>(plan->d_layers, ws, prm);
  RIGL_LAUNCH_CHECK("k_resolve<drop>");
  return RIGL_OK;
}

static int mask_update_launch(rigl_mask_plan* plan, const RunParams& prm_, void* workspace, size_t workspace_bytes,
                              void* stream_) {
  RunParams prm = prm_;
  if (int rc = check_workspace(plan, workspace, workspace_bytes)) return rc;
  RIGL_REQUIRE(prm.grow_mode >= RIGL_GROW_ZEROS && prm.grow_mode <= RIGL_GROW_GRAD_SIGN, "bad grow_mode %d", prm.grow_mode);
  RIGL_REQUIRE(prm.drop_fraction >= 0.f && prm.drop_fraction <= 1.f, "drop_fraction %f outside [0,1]", prm.drop_fraction);
  RIGL_REQUIRE(prm.noise_std >= 0.f, "noise_std must be >= 0");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  if (int rc = launch_drop_select(plan, prm, ws, stream)) return rc;
  k_scan_grow<<<plan->n_blocks, kScanThreads, 0, stream>>>(plan->d_layers, plan->d_tasks, ws, prm);
  RIGL_LAUNCH_CHECK("k_scan_grow");
  k_resolve<true><<<plan->n_layers, kResolveThreads, 0, stream>>>(plan->d_layers, ws, prm);
  RIGL_LAUNCH_CHECK("k_resolve<grow>");
  k_publish_mask<<<plan->n_blocks, kScanThreads, 0, stream>>>(plan->d_layers, plan->d_tasks, ws, prm);
  RIGL_LAUNCH_CHECK("k_publish_mask");
  return RIGL_OK;
}

extern "C" int rigl_mask_update_run(rigl_mask_plan* plan, float drop_fraction, int grow_mode,
                                    float grow_divisor, float acc_scale, int reinit_when_same,
                                    void* workspace, size_t workspace_bytes, void* stream_) {
  RunParams prm{drop_fraction, grow_mode, grow_divisor, acc_scale, reinit_when_same, 0.f, 0u, 0u, 0ull, 0u, 0u};
  return mask_update_launch(plan, prm, workspace, workspace_bytes, stream_);
}

extern "C" int rigl_mask_update_run_noise(rigl_mask_plan* plan, float drop_fraction, int grow_mode,
                                          float grow_divisor, float acc_scale, int reinit_when_same,
                                          float noise_std, uint64_t noise_seed, void* workspace,
                                          size_t workspace_bytes, void* stream_) {
  RunParams prm{drop_fraction, grow_mode, grow_divisor, acc_scale, reinit_when_same, noise_std,
                (uint32_t)(noise_seed & 0xffffffffu), (uint32_t)(noise_seed >> 32), 0ull, 0u, 0u};
  return mask_update_launch(plan, prm, workspace, workspace_bytes, stream_);
}

extern "C" int rigl_mask_prune_run(rigl_mask_plan* plan, const int32_t* keep, const float* old_thr, float* new_thr,
                                   float threshold_decay, void* workspace, size_t workspace_bytes, void* stream_) {
  if (int rc = check_workspace(plan, workspace, workspace_bytes)) return rc;
  RIGL_REQUIRE(keep && old_thr && new_thr, "rigl_mask_prune_run: null keep/old_thr/new_thr");
  RIGL_REQUIRE(threshold_decay >= 0.f && threshold_decay <= 1.f, "threshold_decay %f outside [0,1]", threshold_decay);
  for (int l = 0; l < plan->n_layers; ++l) {
    const LayerDev& L = plan->h_layers[l];
    RIGL_REQUIRE((L.flags & (RIGL_LAYER_DROP_ONLY | RIGL_LAYER_ALL_ACTIVE)) == (RIGL_LAYER_DROP_ONLY | RIGL_LAYER_ALL_ACTIVE)
                     && !L.sdrop && !L.noise,
                 "rigl_mask_prune_run: layer %d needs DROP_ONLY | ALL_ACTIVE, no score_drop and no noise", l);
    RIGL_REQUIRE(keep[l] >= 1 && (uint32_t)keep[l] <= L.n, "rigl_mask_prune_run: layer %d keeps %d of %u", l, keep[l],
                 L.n);
  }
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  // the counts travel as kernel arguments: no copy from host memory, so nothing can wait for the device
  for (int first = 0; first < plan->n_layers; first += kPruneCountBatch) {
    PruneCounts c;
    const int count = std::min(kPruneCountBatch, plan->n_layers - first);
    for (int i = 0; i < count; ++i) c.n_prune[i] = (int32_t)plan->h_layers[first + i].n - keep[first + i];
    k_prune_set_counts<<<1, kScanThreads, 0, stream>>>(plan->d_layers, first, count, c);
    RIGL_LAUNCH_CHECK("k_prune_set_counts");
  }
  RunParams prm{0.f, RIGL_GROW_ZEROS, 1.f, 0.f, 0, 0.f, 0u, 0u, 0ull, 0u, 0u};
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  if (int rc = launch_drop_select(plan, prm, ws, stream)) return rc;
  k_prune_threshold<<<plan->n_layers, kScanThreads, 0, stream>>>(plan->d_layers, ws, old_thr, new_thr, threshold_decay);
  RIGL_LAUNCH_CHECK("k_prune_threshold");
  k_prune_publish<<<plan->n_blocks, kScanThreads, 0, stream>>>(plan->d_layers, plan->d_tasks, new_thr, prm);
  RIGL_LAUNCH_CHECK("k_prune_publish");
  return RIGL_OK;
}

extern "C" int rigl_mask_noise_fill(float* out, int64_t n, uint32_t layer_noise_key, float noise_std,
                                    uint64_t noise_seed, void* stream_) {
  RIGL_REQUIRE(out && n >= 1 && n < (1ll << 31) && noise_std >= 0.f, "rigl_mask_noise_fill: bad arguments");
  RunParams prm{0.f, 0, 1.f, 0.f, 0, noise_std, (uint32_t)(noise_seed & 0xffffffffu), (uint32_t)(noise_seed >> 32), 0ull, 0u, 0u};
  const unsigned blocks = (unsigned)((n + 1023) / 1024);
  k_noise_fill<<<blocks, 256, 0, (cudaStream_t)stream_>>>(out, (uint32_t)n, layer_noise_key, prm);
  RIGL_LAUNCH_CHECK("k_noise_fill");
  return RIGL_OK;
}

extern "C" int rigl_mask_plan_read_stats(const rigl_mask_plan* plan, const void* workspace,
                                         int32_t* out_host, void* stream_) {
  RIGL_REQUIRE(plan && workspace && out_host, "rigl_mask_plan_read_stats: null argument");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  std::vector<LayerState> st(plan->n_layers);
  RIGL_CUDA(cudaMemcpyAsync(st.data(), static_cast<const uint8_t*>(workspace) + plan->state_off,
                            sizeof(LayerState) * plan->n_layers, cudaMemcpyDeviceToHost, stream));
  RIGL_CUDA(cudaStreamSynchronize(stream));
  for (int l = 0; l < plan->n_layers; ++l) {
    const LayerState& s = st[l];
    int32_t* o = out_host + 8 * l;
    o[0] = s.n_ones; o[1] = s.n_prune; o[2] = s.n_keep; o[3] = (int32_t)s.cand_cnt_drop;
    o[4] = (int32_t)s.cand_cnt_grow; o[5] = s.drop_bucket; o[6] = s.grow_bucket; o[7] = 0;
  }
  return RIGL_OK;
}
