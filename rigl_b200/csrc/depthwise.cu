// Depthwise 3x3 convolution (stride 1 / 2, explicit padding 1 = conv2d_fixed_padding) on NHWC bf16 activations:
// forward, input gradient and weight gradient -- HBM-bound streaming kernels.
//
// Replaces depthwise_conv2d_fixed_padding of the reference's MobileNet-v1
// (rigl/imagenet_resnet/mobilenetv1_model.py:120-153, called from mbv1_block_ :186-196).  The depthwise convs are
// NOT masked in the reference (only the pointwise 1x1 convs and the classifier are), but they are a large share of
// the C4 step on the stock cuDNN kernels, so SURVEY 8(f) row 4 ("depthwise") is built as three streaming kernels.
//
// One thread = 8 channels (one 16-byte vector), channels innermost.  Weights: fp32 master [C][1][3][3] (the torch /
// TF depthwise layout flattened as c*9 + kh*3 + kw), rounded to bf16 on load like the activations' compute type;
// fp32 accumulation; bf16 outputs; the weight gradient is fp32, summed in a fixed order (per-CTA partials + a
// finalize pass: deterministic).
#include <cuda_bf16.h>

#include "common.cuh"

namespace rigl {

struct DwGeom {
  int n, h, w, c, oh, ow, s;     // input h x w, output oh x ow, stride s, pad 1, kernel 3
};

__device__ __forceinline__ void dw_unpack8(const uint4& v, float (&f)[8]) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = __bfloat1622float2(h[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ uint4 dw_pack8(const float (&f)[8]) {
  uint4 v;
  __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  return v;
}

// weights of the 8 channels of vector v for tap t, rounded to bf16 (the compute type)
__device__ __forceinline__ void dw_load_w(const float* __restrict__ w, int v, int t, float (&o)[8]) {
#pragma unroll
  for (int e = 0; e < 8; ++e) o[e] = __bfloat162float(__float2bfloat16(__ldg(w + (size_t)(8 * v + e) * 9 + t)));
}

// grid = (column tiles, row groups of kDwRows, images), block = (channel vectors <= 32, columns): no index
// divisions; the 9 x 8 weights of a thread's channel vector are loaded once and reused for its kDwRows pixels.
// FLIP = false: y[n,oh,ow,c] = sum_t x[n, oh*s + kh - 1, ow*s + kw - 1, c] * w[c,kh,kw]
// FLIP = true : dx[n,h,w,c]  = sum_t dy[n, (h + 1 - kh)/s, (w + 1 - kw)/s, c] * w[c,kh,kw]   (where divisible)
constexpr int kDwRows = 8;

template <bool FLIP>
__global__ void __launch_bounds__(256)
k_depthwise3x3(DwGeom g, const __nv_bfloat16* __restrict__ src, const float* __restrict__ w,
               __nv_bfloat16* __restrict__ dst) {
  const int V = g.c >> 3;
  const int out_w = FLIP ? g.w : g.ow, out_h = FLIP ? g.h : g.oh;
  const int in_w = FLIP ? g.ow : g.w, in_h = FLIP ? g.oh : g.h;
  const int col = blockIdx.x * blockDim.y + threadIdx.y, n = blockIdx.z;
  if (col >= out_w) return;
  const int row_end = min(out_h, (int)(blockIdx.y + 1) * kDwRows);
  const bool s2 = g.s == 2;
  for (int v = threadIdx.x; v < V; v += blockDim.x) {
    float wt[9][8];
#pragma unroll
    for (int t = 0; t < 9; ++t) dw_load_w(w, v, t, wt[t]);
    // column taps: source column and validity do not depend on the row
    int wi[3];
    bool wok[3];
#pragma unroll
    for (int kw = 0; kw < 3; ++kw) {
      if (!FLIP) {
        wi[kw] = col * g.s + kw - 1;
        wok[kw] = wi[kw] >= 0 && wi[kw] < in_w;
      } else {
        const int t = col + 1 - kw;
        wok[kw] = t >= 0 && (!s2 || (t & 1) == 0);
        wi[kw] = s2 ? (t >> 1) : t;
        wok[kw] = wok[kw] && wi[kw] < in_w;
      }
      if (!wok[kw]) wi[kw] = 0;                       // clamped: the load stays in bounds, the value is dropped
    }
    const __nv_bfloat16* base = src + (long long)n * in_h * in_w * g.c + 8 * v;
    for (int row = blockIdx.y * kDwRows; row < row_end; ++row) {
      // all nine loads are issued before any arithmetic (no control flow between them: memory-level parallelism)
      uint4 q[9];
      bool ok[9];
#pragma unroll
      for (int kh = 0; kh < 3; ++kh) {
        int hi;
        bool hok;
        if (!FLIP) {
          hi = row * g.s + kh - 1;
          hok = hi >= 0 && hi < in_h;
        } else {
          const int t = row + 1 - kh;
          hok = t >= 0 && (!s2 || (t & 1) == 0);
          hi = s2 ? (t >> 1) : t;
          hok = hok && hi < in_h;
        }
        if (!hok) hi = 0;
#pragma unroll
        for (int kw = 0; kw < 3; ++kw) {
          ok[kh * 3 + kw] = hok && wok[kw];
          q[kh * 3 + kw] = __ldg(reinterpret_cast<const uint4*>(base + ((long long)hi * in_w + wi[kw]) * g.c));
        }
      }
      float acc[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[e] = 0.f;
#pragma unroll
      for (int t = 0; t < 9; ++t) {
        float xs[8];
        dw_unpack8(q[t], xs);
        const float m = ok[t] ? 1.f : 0.f;
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] = fmaf(xs[e] * m, wt[t][e], acc[e]);
      }
      *reinterpret_cast<uint4*>(dst + (((long long)n * out_h + row) * out_w + col) * g.c + 8 * v) = dw_pack8(acc);
    }
  }
}

// Weight gradient: dW[c,kh,kw] = sum over (n, oh, ow) of x[n, oh*s+kh-1, ow*s+kw-1, c] * dy[n,oh,ow,c].
// A CTA owns a contiguous range of output ROWS (n, oh) and ONE group of up to 32 channel vectors; its threads are
// (channel vector, column lane): each accumulates 9 x 8 fp32 sums over its columns of those rows, the column lanes
// are combined through shared memory, and the CTA writes one partial row [9][C-slice].
// block = (bx = min(V, 32) channel vectors, 256 / bx column lanes)
__global__ void __launch_bounds__(256)
k_depthwise3x3_wgrad(DwGeom g, const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy,
                     long long rows_per_block, float* __restrict__ partial /* [gridDim.x][9][C] */) {
  __shared__ float red[256 * 9];                // per element pass: [column lane][vector][tap]
  const int V = g.c >> 3;
  const int bx = blockDim.x, kDwCols = blockDim.y;
  const int v = blockIdx.y * bx + threadIdx.x;  // channel vector of this thread
  const int lane_c = threadIdx.y;               // column lane
  const long long total_rows = (long long)g.n * g.oh;
  const long long r0 = (long long)blockIdx.x * rows_per_block;
  const long long r1 = min(r0 + rows_per_block, total_rows);
  float acc[9][8];
#pragma unroll
  for (int t = 0; t < 9; ++t)
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[t][e] = 0.f;
  if (v < V) {
    for (long long r = r0; r < r1; ++r) {
      const int n = (int)(r / g.oh), oh = (int)(r % g.oh);
      for (int ow = lane_c; ow < g.ow; ow += kDwCols) {
        uint4 q[9];
        bool ok[9];
        const uint4 qd = __ldg(reinterpret_cast<const uint4*>(dy + (((long long)n * g.oh + oh) * g.ow + ow) * g.c + 8 * v));
#pragma unroll
        for (int kh = 0; kh < 3; ++kh) {
          int hi = oh * g.s + kh - 1;
          const bool hok = hi >= 0 && hi < g.h;
          if (!hok) hi = 0;
#pragma unroll
          for (int kw = 0; kw < 3; ++kw) {
            int wi = ow * g.s + kw - 1;
            const bool wok = wi >= 0 && wi < g.w;
            if (!wok) wi = 0;
            ok[kh * 3 + kw] = hok && wok;
            q[kh * 3 + kw] = __ldg(reinterpret_cast<const uint4*>(x + (((long long)n * g.h + hi) * g.w + wi) * g.c + 8 * v));
          }
        }
        float d[8];
        dw_unpack8(qd, d);
#pragma unroll
        for (int t = 0; t < 9; ++t) {
          float xs[8];
          dw_unpack8(q[t], xs);
          const float m = ok[t] ? 1.f : 0.f;
#pragma unroll
          for (int e = 0; e < 8; ++e) acc[t][e] = fmaf(xs[e] * m, d[e], acc[t][e]);
        }
      }
    }
  }
  // combine the column lanes: one of the 8 channel elements at a time through shared memory (fixed order)
  float* out = partial + (size_t)blockIdx.x * 9 * g.c;
#pragma unroll
  for (int e = 0; e < 8; ++e) {                  // (unrolled: acc[][] must stay in registers)
#pragma unroll
    for (int t = 0; t < 9; ++t) red[(lane_c * bx + threadIdx.x) * 9 + t] = acc[t][e];
    __syncthreads();
    if (v < V) {
      for (int t = lane_c; t < 9; t += kDwCols) {     // column lane t sums tap t over all column lanes, fixed order
        float s = 0.f;
        for (int l = 0; l < kDwCols; ++l) s += red[(l * bx + threadIdx.x) * 9 + t];
        out[(size_t)t * g.c + 8 * v + e] = s;
      }
    }
    __syncthreads();
  }
}

// dw[c*9 + t] = beta * dw + sum_b partial[b][t][c]  (fp64 combine, fixed order): block = (32 outputs, 8 slices of b)
__global__ void __launch_bounds__(256)
k_depthwise3x3_wgrad_finalize(const float* __restrict__ partial, int nblocks, int C, float beta,
                              float* __restrict__ dw) {
  __shared__ double sm[8][33];
  const int i = blockIdx.x * 32 + threadIdx.x;                 // i = t * C + c
  double s = 0.0;
  if (i < 9 * C)
    for (int b = threadIdx.y; b < nblocks; b += 8) s += (double)__ldg(partial + (size_t)b * 9 * C + i);
  sm[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y != 0 || i >= 9 * C) return;
  for (int k = 1; k < 8; ++k) s += sm[k][threadIdx.x];
  const int t = i / C, c = i % C;
  float* dst = dw + (size_t)c * 9 + t;
  *dst = (beta != 0.f ? *dst : 0.f) + (float)s;
}

static int dw_geom(int n, int h, int w, int c, int stride, DwGeom* g) {
  RIGL_REQUIRE(n > 0 && h > 0 && w > 0 && c > 0 && c % 8 == 0, "depthwise3x3: channels must be a multiple of 8");
  RIGL_REQUIRE(stride == 1 || stride == 2, "depthwise3x3: stride must be 1 or 2");
  g->n = n; g->h = h; g->w = w; g->c = c; g->s = stride;
  g->oh = (h + 2 - 3) / stride + 1;
  g->ow = (w + 2 - 3) / stride + 1;
  return RIGL_OK;
}

static int dw_wgrad_blocks(const DwGeom& g, long long* rows_per_block) {
  const long long rows = (long long)g.n * g.oh;
  const int V = g.c / 8, bx = V < 32 ? V : 32;
  const int groups = (V + bx - 1) / bx;
  long long target = (kNumSmsHint * 4 + groups - 1) / groups;          // ~4 CTAs per SM in total
  if (target > rows) target = rows;
  if (target < 1) target = 1;
  *rows_per_block = (rows + target - 1) / target;
  return (int)((rows + *rows_per_block - 1) / *rows_per_block);
}

}  // namespace rigl

using namespace rigl;

extern "C" size_t rigl_depthwise3x3_workspace_bytes(int n, int h, int w, int c, int stride) {
  DwGeom g;
  if (dw_geom(n, h, w, c, stride, &g) != RIGL_OK) return 0;
  long long rpb;
  const int nb = dw_wgrad_blocks(g, &rpb);
  return (size_t)nb * 9 * c * sizeof(float) + 256;
}

extern "C" int rigl_depthwise3x3_fprop(const void* x, const float* weights, int n, int h, int w, int c, int stride,
                                       void* y, void* stream) {
  DwGeom g;
  int rc = dw_geom(n, h, w, c, stride, &g);
  if (rc != RIGL_OK) return rc;
  RIGL_REQUIRE(x && weights && y && aligned16(x) && aligned16(y), "rigl_depthwise3x3_fprop: null / unaligned tensor");
  const int V = c / 8, bx = V < 32 ? V : 32, by = 256 / bx;
  dim3 grid((g.ow + by - 1) / by, (g.oh + kDwRows - 1) / kDwRows, g.n), block(bx, by);
  k_depthwise3x3<false><<<grid, block, 0, (cudaStream_t)stream>>>(g, (const __nv_bfloat16*)x, weights, (__nv_bfloat16*)y);
  RIGL_LAUNCH_CHECK("k_depthwise3x3<fprop>");
  return RIGL_OK;
}

extern "C" int rigl_depthwise3x3_dgrad(const void* dy, const float* weights, int n, int h, int w, int c, int stride,
                                       void* dx, void* stream) {
  DwGeom g;
  int rc = dw_geom(n, h, w, c, stride, &g);
  if (rc != RIGL_OK) return rc;
  RIGL_REQUIRE(dy && weights && dx && aligned16(dy) && aligned16(dx), "rigl_depthwise3x3_dgrad: null / unaligned tensor");
  const int V = c / 8, bx = V < 32 ? V : 32, by = 256 / bx;
  dim3 grid((g.w + by - 1) / by, (g.h + kDwRows - 1) / kDwRows, g.n), block(bx, by);
  k_depthwise3x3<true><<<grid, block, 0, (cudaStream_t)stream>>>(g, (const __nv_bfloat16*)dy, weights, (__nv_bfloat16*)dx);
  RIGL_LAUNCH_CHECK("k_depthwise3x3<dgrad>");
  return RIGL_OK;
}

extern "C" int rigl_depthwise3x3_wgrad(const void* x, const void* dy, int n, int h, int w, int c, int stride,
                                       float* dw, float beta, void* ws, size_t ws_bytes, void* stream) {
  DwGeom g;
  int rc = dw_geom(n, h, w, c, stride, &g);
  if (rc != RIGL_OK) return rc;
  RIGL_REQUIRE(x && dy && dw && ws && aligned16(x) && aligned16(dy), "rigl_depthwise3x3_wgrad: null / unaligned tensor");
  RIGL_REQUIRE(beta == 0.f || beta == 1.f, "rigl_depthwise3x3_wgrad: beta must be 0 or 1");
  long long rpb;
  const int nb = dw_wgrad_blocks(g, &rpb);
  float* partial = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(ws) + 255) & ~(uintptr_t)255);
  if (ws_bytes < (size_t)nb * 9 * c * sizeof(float) + 256) {
    set_error("rigl_depthwise3x3_wgrad: workspace too small");
    return RIGL_ERR_WORKSPACE;
  }
  cudaStream_t s = (cudaStream_t)stream;
  const int V = c / 8, bx = V < 32 ? V : 32;       // (V is 4, 8, 16, 32, ... for the MobileNet widths; any V works)
  dim3 grid(nb, (V + bx - 1) / bx), block(bx, 256 / bx);
  k_depthwise3x3_wgrad<<<grid, block, 0, s>>>(g, (const __nv_bfloat16*)x, (const __nv_bfloat16*)dy, rpb, partial);
  RIGL_LAUNCH_CHECK("k_depthwise3x3_wgrad");
  k_depthwise3x3_wgrad_finalize<<<(9 * c + 31) / 32, dim3(32, 8), 0, s>>>(partial, nb, c, beta, dw);
  RIGL_LAUNCH_CHECK("k_depthwise3x3_wgrad_finalize");
  return RIGL_OK;
}
