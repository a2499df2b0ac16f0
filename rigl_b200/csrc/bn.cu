// Fused batch-norm (+ReLU, +residual add) for NHWC bf16 activations -- HBM-bound
// streaming kernels around the masked convs (SURVEY 8f row 1).
//
// Replaces batch_norm_relu (rigl/imagenet_resnet/resnet_model.py:41-80:
// tf.layers.batch_normalization(fused=True, momentum=0.9, epsilon=1e-5) + relu) and the
// `relu(inputs + shortcut)` tail of the bottleneck block (:501).
//
//   forward : stats  : one read of y              -> per-channel mean / rstd (fp32 partials, fp64 combine)
//             apply  : read y (+residual)         -> a = relu(y*scale + shift (+ r)), bf16 (+ 1 bit per element: a > 0)
//   backward: reduce : read da, y (, ReLU bits)   -> dbeta = sum g, dgamma = sum g*xhat  (g = da * relu')
//                      (residual form also writes g, which IS the gradient of the shortcut)
//             apply  : read g|da, y               -> dy = scale * (g - dbeta/M - xhat*dgamma/M)
// MobileNet-v2's linear bottleneck (rigl/imagenet_resnet/mobilenetv2_model.py:246-252) is a BN WITHOUT ReLU, with or
// without an identity shortcut, whose output may have two consumers.  Its residual form stores no ReLU bitmap and its
// backward (column-sum MODE 3) never loads one; a forked plain no-ReLU BN reuses that form with a scratch g.
// Every kernel moves 16-byte vectors (8 channels) per thread with the channel dimension
// innermost, so global traffic is fully coalesced; reductions go registers -> smem ->
// per-block partials -> a tiny finalize kernel (fixed order: deterministic).
// Tensors up to 64 MB take the single-launch variants (k_bn_fwd_fused / k_bn_bwd_fused: the
// same three phases behind two grid barriers); rigl_bn_backward also sums the two gradients of a
// forked block output inside the reduce pass.
#include <cuda_bf16.h>

#include "common.cuh"

namespace rigl {

constexpr int kBnThreads = 256;

__device__ __forceinline__ void unpack8(const uint4& v, float (&f)[8]) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = __bfloat1622float2(h[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  uint4 v;
  __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  return v;
}

// Row grouping of the column-sum pass: vl threads cover the V = C/8 vectors of a row, and one block iteration
// covers rpi rows.  The host sizes the shared memory and the rows per block from the same grouping.
struct RowGroup { int vl, rpi; };
__host__ __device__ __forceinline__ RowGroup row_group(int C, int threads) {
  const int V = C >> 3;
  const int vl = V < threads ? V : threads;
  return {vl, threads / vl};
}

// Column sums of up to two row-wise quantities over a [rows, C] bf16 matrix.
// MODE 0: (y, y^2)                                   -> forward statistics
// MODE 1: (g, g*xhat), g = da * [fma(y,scale,shift) > 0 if relu]      (plain BN / BN+ReLU)
// MODE 2: (g, g*xhat), g = (da [+ da2]) * [relu_bits if relu], g written to gout    (residual form)
// MODE 3: (g, g*xhat), g = da [+ da2], g written to gout     (residual form without ReLU, or a plain no-ReLU BN
//         whose output has two consumers: the linear bottleneck of MobileNet-v2).  Never touches relu_bits.
// partial[block][2][C] fp32.
//
// colsum_vector: this thread's sums (s0, s1) of the 16-byte vector v (channels 8v..8v+7) over rows r0, r0 + step,
// ... < row1.
template <int MODE>
__device__ __forceinline__ void colsum_vector(
    const __nv_bfloat16* __restrict__ y, const __nv_bfloat16* __restrict__ da,
    const __nv_bfloat16* __restrict__ da2, const uint8_t* __restrict__ relu_bits, __nv_bfloat16* __restrict__ gout,
    const float* __restrict__ mean, const float* __restrict__ rstd, const float* __restrict__ scale,
    const float* __restrict__ shift, int relu, long long r0, long long row1, int step, int C, int v, float (&s0)[8],
    float (&s1)[8]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) { s0[i] = 0.f; s1[i] = 0.f; }
  float mu[8], rs[8], sc[8], sh[8];
  if (MODE != 0) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      mu[i] = mean[8 * v + i]; rs[i] = rstd[8 * v + i];
      sc[i] = scale[8 * v + i]; sh[i] = shift[8 * v + i];
    }
  }
  // 4 rows per trip: all loads are issued before any arithmetic (memory-level parallelism)
  for (long long rb = r0; rb < row1; rb += 4ll * step) {
    uint4 qy[4], qd[4], qe[4];
    uint32_t qb[4];
    bool ok[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const long long r = rb + (long long)u * step;
      ok[u] = r < row1;
      if (ok[u]) {
        const long long off = r * C + 8 * v;
        qy[u] = *reinterpret_cast<const uint4*>(y + off);
        if (MODE != 0) qd[u] = *reinterpret_cast<const uint4*>(da + off);
        if (MODE == 2) qb[u] = relu_bits[off >> 3];
        if (MODE >= 2 && da2) qe[u] = *reinterpret_cast<const uint4*>(da2 + off);
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (!ok[u]) continue;
      const long long off = (rb + (long long)u * step) * C + 8 * v;
      float fy[8];
      unpack8(qy[u], fy);
      if (MODE == 0) {
#pragma unroll
        for (int i = 0; i < 8; ++i) { s0[i] += fy[i]; s1[i] = fmaf(fy[i], fy[i], s1[i]); }
      } else {
        float g[8];
        unpack8(qd[u], g);
        if (MODE >= 2) {
          if (da2) {       // the block output feeds two consumers: their gradients are summed here
            float g2[8];   // (rounded to bf16 like the separate elementwise add it replaces)
            unpack8(qe[u], g2);
#pragma unroll
            for (int i = 0; i < 8; ++i) g[i] = __bfloat162float(__float2bfloat16(g[i] + g2[i]));
          }
          if (MODE == 2) {
#pragma unroll
            for (int i = 0; i < 8; ++i) g[i] = (!relu || ((qb[u] >> i) & 1u)) ? g[i] : 0.f;
          }
          *reinterpret_cast<uint4*>(gout + off) = pack8(g);
        } else if (relu) {
#pragma unroll
          for (int i = 0; i < 8; ++i) g[i] = fmaf(fy[i], sc[i], sh[i]) > 0.f ? g[i] : 0.f;
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          s0[i] += g[i];
          s1[i] = fmaf(g[i], (fy[i] - mu[i]) * rs[i], s1[i]);
        }
      }
    }
  }
}

template <int MODE, int THREADS>
__device__ __forceinline__ void colsum_rows(
    const __nv_bfloat16* __restrict__ y, const __nv_bfloat16* __restrict__ da,
    const __nv_bfloat16* __restrict__ da2 /* MODE 2: optional second addend of the output gradient */,
    const uint8_t* __restrict__ relu_bits /* MODE 2 only: bit k of byte i <- forward output [8i+k] > 0 */,
    __nv_bfloat16* __restrict__ gout, const float* __restrict__ mean, const float* __restrict__ rstd,
    const float* __restrict__ scale, const float* __restrict__ shift, int relu, long long row0, long long row1,
    int C, float* __restrict__ partial_row /* [2][C] */, float* red /* smem [rpi][vl][16] */) {
  const int V = C >> 3;                         // 16-byte vectors per row
  const RowGroup grp = row_group(C, THREADS);
  const int vl = grp.vl, rpi = grp.rpi;
  const int r_in = threadIdx.x / vl, v0 = threadIdx.x % vl;
  if (rpi == 1) {
    // V > THREADS / 2: the first vl = min(V, THREADS) threads span one row; when V < THREADS the others have no
    // vector (r_in = 1) and take no part.  Thread v0 owns vectors v0, v0 + vl, ...: their number differs between
    // threads when vl does not divide V (V > THREADS, e.g. C = 2560 at 256 threads), so this loop has no barrier;
    // each thread already holds the whole sums of its vectors.
    if (r_in != 0) return;
    for (int v = v0; v < V; v += vl) {
      float s0[8], s1[8];
      colsum_vector<MODE>(y, da, da2, relu_bits, gout, mean, rstd, scale, shift, relu, row0, row1, 1, C, v, s0, s1);
      float* p0 = partial_row + 8 * v;
#pragma unroll
      for (int i = 0; i < 8; ++i) { p0[i] = s0[i]; p0[C + i] = s1[i]; }
    }
    return;
  }
  // V <= THREADS / 2: one vector per thread (v0), summed by rpi >= 2 row-threads whose sums are combined in shared
  // memory (threads with r_in >= rpi, when vl does not divide THREADS, only join the barriers)
  if (r_in < rpi) {
    float s0[8], s1[8];
    colsum_vector<MODE>(y, da, da2, relu_bits, gout, mean, rstd, scale, shift, relu, row0 + r_in, row1, rpi, C, v0,
                        s0, s1);
    float* dst = red + ((size_t)r_in * vl + v0) * 16;
#pragma unroll
    for (int i = 0; i < 8; ++i) { dst[i] = s0[i]; dst[8 + i] = s1[i]; }
  }
  __syncthreads();
  if (r_in == 0) {
    float a0[8], a1[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { a0[i] = 0.f; a1[i] = 0.f; }
    for (int rr = 0; rr < rpi; ++rr) {
      const float* src = red + ((size_t)rr * vl + v0) * 16;
#pragma unroll
      for (int i = 0; i < 8; ++i) { a0[i] += src[i]; a1[i] += src[8 + i]; }
    }
    float* p0 = partial_row + 8 * v0;
#pragma unroll
    for (int i = 0; i < 8; ++i) { p0[i] = a0[i]; p0[C + i] = a1[i]; }
  }
  __syncthreads();
}


template <int MODE>
__global__ void __launch_bounds__(kBnThreads)
k_bn_colsum(const __nv_bfloat16* __restrict__ y, const __nv_bfloat16* __restrict__ da,
            const __nv_bfloat16* __restrict__ da2, const uint8_t* __restrict__ relu_bits,
            __nv_bfloat16* __restrict__ gout, const float* __restrict__ mean, const float* __restrict__ rstd,
            const float* __restrict__ scale, const float* __restrict__ shift, int relu, long long rows, int C,
            long long rows_per_block, float* __restrict__ partial) {
  extern __shared__ float red[];               // [rpi][V][16]
  const long long row0 = (long long)blockIdx.x * rows_per_block;
  const long long row1 = min(row0 + rows_per_block, rows);
  colsum_rows<MODE, kBnThreads>(y, da, da2, relu_bits, gout, mean, rstd, scale, shift, relu, row0, row1, C,
                                partial + (size_t)blockIdx.x * 2 * C, red);
}

// Sums partial[b][which][c] over b for the CH-channel slab starting at c0, with CH * SLICES threads:
// thread = (channel c0 + t % CH, slice t / CH); slice j adds blocks j, j + SLICES, ... in order, then the slices of a
// warp are combined by shuffles and the warps in warp order.  Every load instruction fetches full 32-byte sectors;
// the reduction is L2-latency bound, so what matters is how many loads are in flight, not bytes.  fp64
// accumulation in a fixed order: deterministic.  The partials may have been written earlier in the same launch,
// so they are read with __ldcg.  Returns true on the threads t < CH whose channel exists, with its sums.
template <int CH, int SLICES>
__device__ __forceinline__ bool slab_sums(const float* partial, int nblocks, int C, int c0, double* s_out,
                                          double* q_out) {
  constexpr int kWarps = CH * SLICES / 32;
  __shared__ double sm_s[kWarps][CH], sm_q[kWarps][CH];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int c = c0 + lane % CH;
  const int slice = warp * (32 / CH) + lane / CH;   // (= threadIdx.x / CH; this form keeps nvcc's 4x loop unroll)
  double s = 0.0, q = 0.0;
  if (c < C) {
    int b = slice;
    for (; b + 3 * SLICES < nblocks; b += 4 * SLICES) {
      float vs[4], vq[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        vs[u] = __ldcg(partial + (size_t)(b + u * SLICES) * 2 * C + c);
        vq[u] = __ldcg(partial + (size_t)(b + u * SLICES) * 2 * C + C + c);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) { s += (double)vs[u]; q += (double)vq[u]; }
    }
    for (; b < nblocks; b += SLICES) {
      s += (double)__ldcg(partial + (size_t)b * 2 * C + c);
      q += (double)__ldcg(partial + (size_t)b * 2 * C + C + c);
    }
  }
#pragma unroll
  for (int o = CH; o < 32; o <<= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    q += __shfl_xor_sync(0xffffffffu, q, o);
  }
  if (lane < CH) { sm_s[warp][lane] = s; sm_q[warp][lane] = q; }
  __syncthreads();
  if (threadIdx.x >= CH) return false;
  s = 0.0; q = 0.0;
  for (int w = 0; w < kWarps; ++w) { s += sm_s[w][threadIdx.x]; q += sm_q[w][threadIdx.x]; }
  *s_out = s; *q_out = q;
  return c < C;
}

// Forward finalize of channel c from its sums (s, q) of y and y^2 over `rows`: mean, rstd, scale = gamma*rstd,
// shift = beta - mean*scale, running stats.
__device__ __forceinline__ void finalize_fwd_channel(int c, double s, double q, long long rows, float eps,
                                                     float momentum, const float* __restrict__ gamma,
                                                     const float* __restrict__ beta, float* mean, float* rstd,
                                                     float* scale, float* shift, float* __restrict__ running_mean,
                                                     float* __restrict__ running_var) {
  const double m = s / (double)rows;
  double var = q / (double)rows - m * m;
  if (var < 0.0) var = 0.0;
  const float r = (float)(1.0 / sqrt(var + (double)eps));
  mean[c] = (float)m;
  rstd[c] = r;
  const float sc = gamma[c] * r;
  scale[c] = sc;
  shift[c] = beta[c] - (float)m * sc;
  if (running_mean) {
    const double unbiased = rows > 1 ? var * (double)rows / (double)(rows - 1) : var;
    running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * (float)m;
    running_var[c] = (1.f - momentum) * running_var[c] + momentum * (float)unbiased;
  }
}

// Backward finalize of channel c from its sums (s, q) of g and g*xhat: dbeta, dgamma and the per-channel affine
// form of the input gradient
//   dy = scale*g + P*y + Q,  P = -scale*rstd*dgamma/M,  Q = scale*(rstd*mean*dgamma/M - dbeta/M).
__device__ __forceinline__ void finalize_bwd_channel(int c, double s, double q, long long rows, int C,
                                                     const float* __restrict__ mean, const float* __restrict__ rstd,
                                                     const float* __restrict__ scale, float* __restrict__ dgamma,
                                                     float* __restrict__ dbeta, float* coef /*[2][C]: P, Q*/) {
  dbeta[c] = (float)s;
  dgamma[c] = (float)q;
  const double c0 = s / (double)rows, c1 = q / (double)rows;
  const double sc = (double)scale[c], r = (double)rstd[c], m = (double)mean[c];
  coef[c] = (float)(-sc * r * c1);
  coef[C + c] = (float)(sc * (r * m * c1 - c0));
}

// One 1024-thread CTA per 8 channels (the reduction is L2-latency bound: many loads in flight per channel).
constexpr int kFinCh = 8, kFinSlices = 128;

__global__ void __launch_bounds__(kFinCh * kFinSlices)
k_bn_finalize_fwd(const float* __restrict__ partial, int nblocks, int C, long long rows, float eps,
                  const float* __restrict__ gamma, const float* __restrict__ beta, float* __restrict__ mean,
                  float* __restrict__ rstd, float* __restrict__ scale, float* __restrict__ shift,
                  float* __restrict__ running_mean, float* __restrict__ running_var, float momentum) {
  double s, q;
  if (!slab_sums<kFinCh, kFinSlices>(partial, nblocks, C, blockIdx.x * kFinCh, &s, &q)) return;
  finalize_fwd_channel(blockIdx.x * kFinCh + threadIdx.x, s, q, rows, eps, momentum, gamma, beta, mean, rstd, scale,
                       shift, running_mean, running_var);
}

__global__ void __launch_bounds__(kFinCh * kFinSlices)
k_bn_finalize_bwd(const float* __restrict__ partial, int nblocks, int C, long long rows,
                  const float* __restrict__ mean, const float* __restrict__ rstd, const float* __restrict__ scale,
                  float* __restrict__ dgamma, float* __restrict__ dbeta, float* __restrict__ coef) {
  double s, q;
  if (!slab_sums<kFinCh, kFinSlices>(partial, nblocks, C, blockIdx.x * kFinCh, &s, &q)) return;
  finalize_bwd_channel(blockIdx.x * kFinCh + threadIdx.x, s, q, rows, C, mean, rstd, scale, dgamma, dbeta, coef);
}

// Forward apply of one vector held in registers: a = [relu](f*sc + sh (+ r if has_r)).  Returns a packed to
// bf16; *bits <- which outputs are positive (all the residual backward needs of this tensor).
__device__ __forceinline__ uint4 bn_apply8(float (&f)[8], const float (&sc)[8], const float (&sh)[8],
                                           const float (&r)[8], bool has_r, int relu, uint32_t* bits) {
#pragma unroll
  for (int k = 0; k < 8; ++k) f[k] = fmaf(f[k], sc[k], sh[k]);
  if (has_r) {
#pragma unroll
    for (int k = 0; k < 8; ++k) f[k] += r[k];
  }
  if (relu) {
#pragma unroll
    for (int k = 0; k < 8; ++k) f[k] = fmaxf(f[k], 0.f);
  }
  uint32_t m = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) m |= (f[k] > 0.f ? 1u : 0u) << k;
  *bits = m;
  return pack8(f);
}

// Backward apply of one vector held in registers: dy = sc*g + P*y + Q, with g zeroed where the ReLU was inactive
// when relu_recompute (the mask recomputed from y; otherwise g arrives masked).
__device__ __forceinline__ uint4 bn_bwd_apply8(float (&g)[8], const float (&fy)[8], const float (&sc)[8],
                                               const float (&sh)[8], const float (&P)[8], const float (&Q)[8],
                                               bool relu_recompute) {
  if (relu_recompute) {
#pragma unroll
    for (int k = 0; k < 8; ++k)
      if (!(fmaf(fy[k], sc[k], sh[k]) > 0.f)) g[k] = 0.f;
  }
  float o[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) o[k] = fmaf(sc[k], g[k], fmaf(P[k], fy[k], Q[k]));
  return pack8(o);
}

__device__ __forceinline__ void load8f(const float* __restrict__ p, int v, float (&o)[8]) {
  const float4 a = reinterpret_cast<const float4*>(p)[2 * v], b = reinterpret_cast<const float4*>(p)[2 * v + 1];
  o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.w; o[4] = b.x; o[5] = b.y; o[6] = b.z; o[7] = b.w;
}

// a = [relu](y*scale + shift (+ residual)).  The grid stride is a multiple of V whenever V
// divides the thread count, so each thread keeps ONE channel vector: its coefficients are
// loaded once and the loop only streams activations.
__global__ void __launch_bounds__(kBnThreads)
k_bn_apply(const __nv_bfloat16* __restrict__ y, const __nv_bfloat16* __restrict__ residual,
           const float* __restrict__ scale, const float* __restrict__ shift, int relu, long long nvec, int V,
           __nv_bfloat16* __restrict__ out, uint8_t* __restrict__ relu_bits) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long i0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const bool fixed_v = (stride % V) == 0;
  float sc[8], sh[8];
  if (fixed_v) { load8f(scale, (int)(i0 % V), sc); load8f(shift, (int)(i0 % V), sh); }
  for (long long i = i0; i < nvec; i += stride) {
    if (!fixed_v) { load8f(scale, (int)(i % V), sc); load8f(shift, (int)(i % V), sh); }
    float f[8], r[8];
    unpack8(reinterpret_cast<const uint4*>(y)[i], f);
    uint32_t m;
    uint4 a;
    if (residual) {   // one call per case: a single call with a run-time flag costs this kernel 8 more registers
      unpack8(reinterpret_cast<const uint4*>(residual)[i], r);
      a = bn_apply8(f, sc, sh, r, true, relu, &m);
    } else {
      a = bn_apply8(f, sc, sh, r, false, relu, &m);
    }
    reinterpret_cast<uint4*>(out)[i] = a;
    if (relu_bits) relu_bits[i] = (uint8_t)m;
  }
}

// dy = scale*g + P*y + Q;  g = da * relu' (recomputed from y) or the stored g.
__global__ void __launch_bounds__(kBnThreads)
k_bn_bwd_apply(const __nv_bfloat16* __restrict__ g_or_da, const __nv_bfloat16* __restrict__ y,
               const float* __restrict__ scale, const float* __restrict__ shift, const float* __restrict__ coef,
               int relu_recompute, long long nvec, int V, int C, __nv_bfloat16* __restrict__ dy) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long i0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const bool fixed_v = (stride % V) == 0;
  float sc[8], sh[8], P[8], Q[8];
  if (fixed_v) {
    const int v = (int)(i0 % V);
    load8f(scale, v, sc); load8f(shift, v, sh); load8f(coef, v, P); load8f(coef + C, v, Q);
  }
  for (long long i = i0; i < nvec; i += stride) {
    if (!fixed_v) {
      const int v = (int)(i % V);
      load8f(scale, v, sc); load8f(shift, v, sh); load8f(coef, v, P); load8f(coef + C, v, Q);
    }
    float g[8], fy[8];
    unpack8(reinterpret_cast<const uint4*>(g_or_da)[i], g);
    unpack8(reinterpret_cast<const uint4*>(y)[i], fy);
    reinterpret_cast<uint4*>(dy)[i] = bn_bwd_apply8(g, fy, sc, sh, P, Q, relu_recompute != 0);
  }
}


// ----------------------------------------------------------------------------
// Single-launch variants for tensors up to g_bn_fused_max_bytes (64 MB: 40 of ResNet-50's 53 BNs at batch 256
// move <= 51 MB).  The three passes of a direction (column sums -> finalize -> apply) become three phases of ONE
// persistent kernel separated by grid barriers: two dependent launch boundaries disappear, and the apply phase
// re-reads the rows this CTA just summed, from L2 where they still fit.  H100's 50 MB of L2 does not hold the
// largest of these tensors, and the 64 MB cutoff has not been re-measured there (tools/bench_bn_layer.py compares
// the two paths per size; RIGL_BN_FUSED=0 selects the three-kernel path).  Both paths call the same column-sum,
// finalize and per-vector apply functions and sum the per-CTA partials in CTA order, so results are bit-identical
// to the three-kernel path run with the same grid.  Data written earlier in the same launch (partials, scale /
// shift, coef) is read with __ldcg, never through a non-coherent load.  All CTAs must be co-resident
// (grid <= occupancy x SMs, checked by the host).
// ----------------------------------------------------------------------------
constexpr int kFusedThreads = 512;
constexpr int kFusedCh = 32, kFusedSlices = kFusedThreads / kFusedCh;   // finalize: 32 channels per CTA

struct BnSync { unsigned int arrived; unsigned int done; };

__device__ __forceinline__ void grid_barrier(BnSync* sync, unsigned int target) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(&sync->arrived, 1u);
    unsigned int v, spins = 0;
    long long t0 = 0;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(&sync->arrived) : "memory");
      if (v < target && (++spins & 0x3FFu) == 0) {        // a CTA that never arrives (grid not co-resident) must
        const long long now = clock64();                   // not hang the GPU: trap after ~2 s
        if (t0 == 0) t0 = now;
        else if (now - t0 > 4000000000ll) __trap();
      }
    } while (v < target);
    __threadfence();
  }
  __syncthreads();
}
// The last CTA to finish re-arms the counters for the next launch (every CTA has left both barriers by then).
__device__ __forceinline__ void grid_barrier_release(BnSync* sync) {
  __syncthreads();
  if (threadIdx.x == 0) {
    if (atomicAdd(&sync->done, 1u) == gridDim.x - 1) {
      sync->arrived = 0u;
      sync->done = 0u;
      __threadfence();
    }
  }
}

__global__ void __launch_bounds__(kFusedThreads, 1)
k_bn_fwd_fused(const __nv_bfloat16* __restrict__ y, const __nv_bfloat16* __restrict__ residual,
               const float* __restrict__ gamma, const float* __restrict__ beta, long long rows, int C,
               long long rows_per_block, float eps, float momentum, int relu, float* __restrict__ running_mean,
               float* __restrict__ running_var, float* mean, float* rstd, float* scale, float* shift,
               __nv_bfloat16* __restrict__ out, float* partial, BnSync* sync, uint8_t* __restrict__ relu_bits) {
  extern __shared__ float red[];
  const long long row0 = min((long long)blockIdx.x * rows_per_block, rows);
  const long long row1 = min(row0 + rows_per_block, rows);
  // ---- phase 1: column sums of this CTA's rows
  colsum_rows<0, kFusedThreads>(y, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, 0, row0, row1,
                                C, partial + (size_t)blockIdx.x * 2 * C, red);
  grid_barrier(sync, gridDim.x);
  // ---- phase 2: mean / rstd / scale / shift, 32 channels per CTA
  for (int slab = blockIdx.x; slab * kFusedCh < C; slab += gridDim.x) {
    double s, q;
    if (slab_sums<kFusedCh, kFusedSlices>(partial, gridDim.x, C, slab * kFusedCh, &s, &q))
      finalize_fwd_channel(slab * kFusedCh + threadIdx.x, s, q, rows, eps, momentum, gamma, beta, mean, rstd, scale,
                           shift, running_mean, running_var);
    __syncthreads();
  }
  grid_barrier(sync, 2 * gridDim.x);
  // ---- phase 3: apply to the same rows (L2-resident)
  {
    const int V = C >> 3;
    const long long i_end = row1 * V;
    const bool fixed_v = (kFusedThreads % V) == 0;
    float sc[8], sh[8];
    long long i = row0 * V + threadIdx.x;
    if (fixed_v && i < i_end) {
      const int v = (int)(i % V);
#pragma unroll
      for (int k = 0; k < 8; ++k) { sc[k] = __ldcg(scale + 8 * v + k); sh[k] = __ldcg(shift + 8 * v + k); }
    }
    // 4 vectors in flight per thread (each thread walks ~20 vectors: one at a time is latency bound)
    for (; i < i_end; i += 4ll * kFusedThreads) {
      uint4 qy[4], qr[4];
      bool ok[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const long long idx = i + (long long)u * kFusedThreads;
        ok[u] = idx < i_end;
        if (ok[u]) {
          qy[u] = reinterpret_cast<const uint4*>(y)[idx];
          if (residual) qr[u] = reinterpret_cast<const uint4*>(residual)[idx];
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (!ok[u]) continue;
        const long long idx = i + (long long)u * kFusedThreads;
        if (!fixed_v) {
          const int v = (int)(idx % V);
#pragma unroll
          for (int k = 0; k < 8; ++k) { sc[k] = __ldcg(scale + 8 * v + k); sh[k] = __ldcg(shift + 8 * v + k); }
        }
        float f[8], r[8];
        unpack8(qy[u], f);
        if (residual) unpack8(qr[u], r);
        uint32_t m;
        reinterpret_cast<uint4*>(out)[idx] = bn_apply8(f, sc, sh, r, residual != nullptr, relu, &m);
        if (relu_bits) relu_bits[idx] = (uint8_t)m;
      }
    }
  }
  grid_barrier_release(sync);
}

template <int MODE>
__global__ void __launch_bounds__(kFusedThreads, 1)
k_bn_bwd_fused(const __nv_bfloat16* __restrict__ da, const __nv_bfloat16* __restrict__ da2,
               const __nv_bfloat16* __restrict__ y, const uint8_t* __restrict__ relu_bits,
               const float* __restrict__ mean, const float* __restrict__ rstd, const float* __restrict__ scale,
               const float* __restrict__ shift, long long rows, int C, long long rows_per_block, int relu,
               __nv_bfloat16* __restrict__ dy, __nv_bfloat16* gout, float* __restrict__ dgamma,
               float* __restrict__ dbeta, float* partial, float* coef, BnSync* sync) {
  extern __shared__ float red[];
  const long long row0 = min((long long)blockIdx.x * rows_per_block, rows);
  const long long row1 = min(row0 + rows_per_block, rows);
  colsum_rows<MODE, kFusedThreads>(y, da, da2, relu_bits, gout, mean, rstd, scale, shift, relu, row0, row1, C,
                                   partial + (size_t)blockIdx.x * 2 * C, red);
  grid_barrier(sync, gridDim.x);
  for (int slab = blockIdx.x; slab * kFusedCh < C; slab += gridDim.x) {
    double s, q;
    if (slab_sums<kFusedCh, kFusedSlices>(partial, gridDim.x, C, slab * kFusedCh, &s, &q))
      finalize_bwd_channel(slab * kFusedCh + threadIdx.x, s, q, rows, C, mean, rstd, scale, dgamma, dbeta, coef);
    __syncthreads();
  }
  grid_barrier(sync, 2 * gridDim.x);
  {
    const int V = C >> 3;
    const long long i_end = row1 * V;
    const bool fixed_v = (kFusedThreads % V) == 0;
    const __nv_bfloat16* g_src = (MODE >= 2) ? gout : da;      // (gout was written by THIS CTA for these rows)
    float sc[8], sh[8], P[8], Q[8];
    long long i = row0 * V + threadIdx.x;
    auto load_coef = [&](int v) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        sc[k] = scale[8 * v + k]; sh[k] = shift[8 * v + k];
        P[k] = __ldcg(coef + 8 * v + k); Q[k] = __ldcg(coef + C + 8 * v + k);
      }
    };
    if (fixed_v && i < i_end) load_coef((int)(i % V));
    for (; i < i_end; i += 4ll * kFusedThreads) {
      uint4 qg[4], qy[4];
      bool ok[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const long long idx = i + (long long)u * kFusedThreads;
        ok[u] = idx < i_end;
        if (ok[u]) {
          qg[u] = reinterpret_cast<const uint4*>(g_src)[idx];
          qy[u] = reinterpret_cast<const uint4*>(y)[idx];
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (!ok[u]) continue;
        const long long idx = i + (long long)u * kFusedThreads;
        if (!fixed_v) load_coef((int)(idx % V));
        float g[8], fy[8];
        unpack8(qg[u], g);
        unpack8(qy[u], fy);
        reinterpret_cast<uint4*>(dy)[idx] = bn_bwd_apply8(g, fy, sc, sh, P, Q, MODE == 1 && relu);
      }
    }
  }
  grid_barrier_release(sync);
}

static bool g_bn_fused = true;            // RIGL_BN_FUSED=0: always the 3-kernel path
static size_t g_bn_fused_max_bytes = (size_t)64 << 20;
static BnSync* g_bn_sync[16] = {};
static int g_bn_fused_grid[4] = {0, 0, 0, 0};   // co-resident CTAs: fwd, bwd<1>, bwd<2>, bwd<3> (0 = not probed)

// Dynamic shared memory of the column-sum pass: [rpi][vl][16] floats.
static size_t colsum_smem(int C, int threads) {
  const RowGroup grp = row_group(C, threads);
  return (size_t)grp.rpi * grp.vl * 16 * sizeof(float);
}

// Rows per CTA for about `target` CTAs: a multiple of the rows one block iteration covers.
static long long rows_per_block(long long rows, int C, int threads, long long target) {
  const int rpi = row_group(C, threads).rpi;
  long long rpb = (rows + target - 1) / target;
  rpb = (rpb + rpi - 1) / rpi * rpi;
  return rpb < rpi ? rpi : rpb;
}

// Grid (<= co-resident capacity) and rows per CTA of the fused kernels; 0 = use the 3-kernel path.
static int fused_plan(int which, long long rows, int C, long long* rows_per_blk, BnSync** sync) {
  static bool env_read = false;
  if (!env_read) {
    if (const char* e = getenv("RIGL_BN_FUSED")) g_bn_fused = !(e[0] == '0');
    env_read = true;
  }
  if (!g_bn_fused || C % 8 || C > 4096 || (size_t)rows * C * 2 > g_bn_fused_max_bytes) return 0;
  // (tools/bench_bn_layer.py compares the two: the backward wins at every size <= 64 MB, the forward only
  //  for wide layers -- with few vectors per row the one-block-per-SM 512-thread grid hides less latency than 3
  //  big grids)
  if (which == 0 && C < 512) return 0;
  if (colsum_smem(C, kFusedThreads) > 32 * 1024) return 0;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 16) return 0;
  if (g_bn_fused_grid[which] == 0) {
    int sms = 0, per_sm = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaError_t e = cudaSuccess;
    if (which == 0) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_bn_fwd_fused, kFusedThreads, 32 * 1024);
    else if (which == 1) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_bn_bwd_fused<1>, kFusedThreads, 32 * 1024);
    else if (which == 2) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_bn_bwd_fused<2>, kFusedThreads, 32 * 1024);
    else e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_bn_bwd_fused<3>, kFusedThreads, 32 * 1024);
    if (e != cudaSuccess || per_sm < 1) { g_bn_fused_grid[which] = -1; return 0; }
    if (per_sm > 2) per_sm = 2;
    g_bn_fused_grid[which] = sms * per_sm;
  }
  if (g_bn_fused_grid[which] < 0) return 0;
  if (g_bn_sync[dev] == nullptr) {
    if (cudaMalloc(&g_bn_sync[dev], 4 * sizeof(BnSync)) != cudaSuccess) return 0;
    cudaMemset(g_bn_sync[dev], 0, 4 * sizeof(BnSync));
  }
  const long long rpb = rows_per_block(rows, C, kFusedThreads, g_bn_fused_grid[which]);
  *rows_per_blk = rpb;
  *sync = g_bn_sync[dev] + which;
  return (int)((rows + rpb - 1) / rpb);
}

static int colsum_blocks(long long rows, int C, long long* rows_per_blk) {
  const long long rpb = rows_per_block(rows, C, kBnThreads, kNumSmsHint * 6);   // ~6 resident blocks per SM
  *rows_per_blk = rpb;
  return (int)((rows + rpb - 1) / rpb);
}

// Grid of the grid-stride apply kernels.
static unsigned apply_blocks(long long nvec) {
  const long long blocks = (nvec + kBnThreads - 1) / kBnThreads;
  return (unsigned)(blocks > kNumSmsHint * 16 ? kNumSmsHint * 16 : blocks);
}

static int launch_bn_apply(const void* y, const void* residual, const float* scale, const float* shift, int relu,
                           long long rows, int channels, void* out, void* relu_bits, cudaStream_t s) {
  const long long nvec = rows * (channels / 8);
  k_bn_apply<<<apply_blocks(nvec), kBnThreads, 0, s>>>((const __nv_bfloat16*)y, (const __nv_bfloat16*)residual,
                                                       scale, shift, relu, nvec, channels / 8, (__nv_bfloat16*)out,
                                                       static_cast<uint8_t*>(relu_bits));
  RIGL_LAUNCH_CHECK("k_bn_apply");
  return RIGL_OK;
}

}  // namespace rigl

using namespace rigl;

extern "C" size_t rigl_bn_workspace_bytes(int64_t rows, int channels) {
  if (rows <= 0 || channels <= 0) return 0;
  long long rpb;
  const int nb = colsum_blocks(rows, channels, &rpb);
  return (size_t)nb * 2 * channels * sizeof(float) + 256;
}

extern "C" int rigl_bn_forward_train(const void* y, const void* residual, const float* gamma, const float* beta,
                                     int64_t rows, int channels, float eps, float momentum, int relu,
                                     float* running_mean, float* running_var, float* save_mean, float* save_rstd,
                                     float* save_scale, float* save_shift, void* out, void* ws, size_t ws_bytes,
                                     void* relu_bits, void* stream_) {
  RIGL_REQUIRE(y && gamma && beta && save_mean && save_rstd && save_scale && save_shift && out && ws,
               "rigl_bn_forward_train: null argument");
  RIGL_REQUIRE(rows > 0 && channels > 0 && channels % 8 == 0, "rigl_bn_forward_train: channels must be a multiple of 8");
  RIGL_REQUIRE(aligned16(y) && aligned16(out) && aligned16(residual) && aligned16(save_scale) && aligned16(save_shift),
               "rigl_bn_forward_train: tensors must be 16-byte aligned");
  cudaStream_t s = (cudaStream_t)stream_;
  {
    BnSync* sync = nullptr;
    long long frpb;
    const int grid = fused_plan(0, rows, channels, &frpb, &sync);
    if (grid > 0 && ws_bytes >= (size_t)grid * 2 * channels * sizeof(float)) {
      k_bn_fwd_fused<<<grid, kFusedThreads, colsum_smem(channels, kFusedThreads), s>>>(
          (const __nv_bfloat16*)y, (const __nv_bfloat16*)residual, gamma, beta, rows, channels, frpb, eps, momentum, relu,
          running_mean, running_var, save_mean, save_rstd, save_scale, save_shift, (__nv_bfloat16*)out,
          static_cast<float*>(ws), sync, static_cast<uint8_t*>(relu_bits));
      RIGL_LAUNCH_CHECK("k_bn_fwd_fused");
      return RIGL_OK;
    }
  }
  long long rpb;
  const int nb = colsum_blocks(rows, channels, &rpb);
  if (ws_bytes < (size_t)nb * 2 * channels * sizeof(float)) {
    set_error("rigl_bn_forward_train: workspace too small");
    return RIGL_ERR_WORKSPACE;
  }
  float* partial = static_cast<float*>(ws);
  k_bn_colsum<0><<<nb, kBnThreads, colsum_smem(channels, kBnThreads), s>>>(
      (const __nv_bfloat16*)y, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, 0, rows, channels,
      rpb, partial);
  RIGL_LAUNCH_CHECK("k_bn_colsum<0>");
  return rigl_bn_forward_train_partials(y, residual, gamma, beta, partial, nb, rows, channels, eps, momentum, relu,
                                        running_mean, running_var, save_mean, save_rstd, save_scale, save_shift, out,
                                        relu_bits, stream_);
}

// Same as rigl_bn_forward_train but the column sums come from the producing conv's epilogue
// (partial[rows][2][channels], as written by rigl_masked_conv2d_fprop_bnstats): no stats pass.
extern "C" int rigl_bn_forward_train_partials(const void* y, const void* residual, const float* gamma,
                                              const float* beta, const float* partial, int partial_rows,
                                              int64_t rows, int channels, float eps, float momentum, int relu,
                                              float* running_mean, float* running_var, float* save_mean,
                                              float* save_rstd, float* save_scale, float* save_shift, void* out,
                                              void* relu_bits, void* stream_) {
  RIGL_REQUIRE(y && gamma && beta && partial && save_mean && save_rstd && save_scale && save_shift && out,
               "rigl_bn_forward_train_partials: null argument");
  RIGL_REQUIRE(rows > 0 && channels > 0 && channels % 8 == 0 && partial_rows > 0,
               "rigl_bn_forward_train_partials: bad sizes");
  cudaStream_t s = (cudaStream_t)stream_;
  k_bn_finalize_fwd<<<(channels + kFinCh - 1) / kFinCh, kFinCh * kFinSlices, 0, s>>>(
      partial, partial_rows, channels, rows, eps, gamma, beta, save_mean, save_rstd, save_scale, save_shift,
      running_mean, running_var, momentum);
  RIGL_LAUNCH_CHECK("k_bn_finalize_fwd");
  return launch_bn_apply(y, residual, save_scale, save_shift, relu, rows, channels, out, relu_bits, s);
}

extern "C" int rigl_bn_apply(const void* y, const void* residual, const float* scale, const float* shift,
                             int64_t rows, int channels, int relu, void* out, void* stream_) {
  RIGL_REQUIRE(y && scale && shift && out && rows > 0 && channels > 0 && channels % 8 == 0,
               "rigl_bn_apply: bad arguments");
  return launch_bn_apply(y, residual, scale, shift, relu, rows, channels, out, nullptr, (cudaStream_t)stream_);
}

extern "C" int rigl_bn_backward(const void* da, const void* da2, const void* y, const float* save_mean,
                                const float* save_rstd, const float* save_scale, const float* save_shift,
                                int64_t rows, int channels, int relu, void* dy, void* dresidual, float* dgamma,
                                float* dbeta, void* ws, size_t ws_bytes, const void* relu_bits, void* stream_) {
  RIGL_REQUIRE(da2 == nullptr || (dresidual != nullptr && aligned16(da2)),
               "rigl_bn_backward: a second output gradient needs the residual form (dresidual != NULL)");
  RIGL_REQUIRE(da && y && save_mean && save_rstd && save_scale && save_shift && dy && dgamma && dbeta && ws,
               "rigl_bn_backward: null argument");
  RIGL_REQUIRE(rows > 0 && channels > 0 && channels % 8 == 0, "rigl_bn_backward: channels must be a multiple of 8");
  RIGL_REQUIRE(dresidual == nullptr || !relu || relu_bits != nullptr,
               "rigl_bn_backward: the residual form with a ReLU needs the ReLU bitmap written by the forward pass");
  cudaStream_t s = (cudaStream_t)stream_;
  const bool residual_form = dresidual != nullptr;
  // 1: plain (da, recomputed ReLU mask); 2: residual with ReLU (stored bitmap); 3: residual / forked without ReLU
  const int mode = !residual_form ? 1 : relu ? 2 : 3;
  {
    BnSync* sync = nullptr;
    long long frpb;
    const int grid = fused_plan(mode, rows, channels, &frpb, &sync);
    if (grid > 0 && ws_bytes >= ((size_t)grid * 2 * channels + 2 * channels) * sizeof(float)) {
      float* partial = static_cast<float*>(ws);
      float* coef = partial + (size_t)grid * 2 * channels;
      if (mode == 2) {
        k_bn_bwd_fused<2><<<grid, kFusedThreads, colsum_smem(channels, kFusedThreads), s>>>(
            (const __nv_bfloat16*)da, (const __nv_bfloat16*)da2, (const __nv_bfloat16*)y,
            static_cast<const uint8_t*>(relu_bits), save_mean, save_rstd, save_scale, save_shift, rows, channels, frpb,
            relu, (__nv_bfloat16*)dy, (__nv_bfloat16*)dresidual, dgamma, dbeta, partial, coef, sync);
      } else if (mode == 3) {
        k_bn_bwd_fused<3><<<grid, kFusedThreads, colsum_smem(channels, kFusedThreads), s>>>(
            (const __nv_bfloat16*)da, (const __nv_bfloat16*)da2, (const __nv_bfloat16*)y, nullptr, save_mean,
            save_rstd, save_scale, save_shift, rows, channels, frpb, 0, (__nv_bfloat16*)dy, (__nv_bfloat16*)dresidual,
            dgamma, dbeta, partial, coef, sync);
      } else {
        k_bn_bwd_fused<1><<<grid, kFusedThreads, colsum_smem(channels, kFusedThreads), s>>>(
            (const __nv_bfloat16*)da, nullptr, (const __nv_bfloat16*)y, nullptr, save_mean, save_rstd, save_scale,
            save_shift, rows, channels, frpb, relu, (__nv_bfloat16*)dy, nullptr, dgamma, dbeta, partial, coef, sync);
      }
      RIGL_LAUNCH_CHECK("k_bn_bwd_fused");
      return RIGL_OK;
    }
  }
  long long rpb;
  const int nb = colsum_blocks(rows, channels, &rpb);
  const size_t need = (size_t)nb * 2 * channels * sizeof(float) + 2 * channels * sizeof(float);
  if (ws_bytes < need) {
    set_error("rigl_bn_backward: workspace too small");
    return RIGL_ERR_WORKSPACE;
  }
  float* partial = static_cast<float*>(ws);
  float* coef = partial + (size_t)nb * 2 * channels;
  if (mode == 2) {
    k_bn_colsum<2><<<nb, kBnThreads, colsum_smem(channels, kBnThreads), s>>>(
        (const __nv_bfloat16*)y, (const __nv_bfloat16*)da, (const __nv_bfloat16*)da2,
        static_cast<const uint8_t*>(relu_bits), (__nv_bfloat16*)dresidual, save_mean, save_rstd, save_scale,
        save_shift, relu, rows, channels, rpb, partial);
    RIGL_LAUNCH_CHECK("k_bn_colsum<2>");
  } else if (mode == 3) {
    k_bn_colsum<3><<<nb, kBnThreads, colsum_smem(channels, kBnThreads), s>>>(
        (const __nv_bfloat16*)y, (const __nv_bfloat16*)da, (const __nv_bfloat16*)da2, nullptr,
        (__nv_bfloat16*)dresidual, save_mean, save_rstd, save_scale, save_shift, 0, rows, channels, rpb, partial);
    RIGL_LAUNCH_CHECK("k_bn_colsum<3>");
  } else {
    k_bn_colsum<1><<<nb, kBnThreads, colsum_smem(channels, kBnThreads), s>>>(
        (const __nv_bfloat16*)y, (const __nv_bfloat16*)da, nullptr, nullptr, nullptr, save_mean, save_rstd, save_scale,
        save_shift, relu, rows, channels, rpb, partial);
    RIGL_LAUNCH_CHECK("k_bn_colsum<1>");
  }
  k_bn_finalize_bwd<<<(channels + kFinCh - 1) / kFinCh, kFinCh * kFinSlices, 0, s>>>(
      partial, nb, channels, rows, save_mean, save_rstd, save_scale, dgamma, dbeta, coef);
  RIGL_LAUNCH_CHECK("k_bn_finalize_bwd");
  const long long nvec = rows * (channels / 8);
  k_bn_bwd_apply<<<apply_blocks(nvec), kBnThreads, 0, s>>>(
      (const __nv_bfloat16*)(residual_form ? dresidual : da), (const __nv_bfloat16*)y, save_scale, save_shift, coef,
      (!residual_form && relu) ? 1 : 0, nvec, channels / 8, channels, (__nv_bfloat16*)dy);
  RIGL_LAUNCH_CHECK("k_bn_bwd_apply");
  return RIGL_OK;
}
