// Max pooling for NHWC bf16 activations (the stem's 3x3/2 pool), HBM-bound streaming kernels.
// Replaces tf.layers.max_pooling2d(pool_size=3, strides=2, padding='SAME')
// (rigl/imagenet_resnet/resnet_model.py:636-642) with TF's SAME rule: pad_total =
// max((out-1)*s + k - in, 0), pad_before = pad_total / 2 (so 112 -> 56 pads only at the end).
// Forward stores the window-relative argmax (first maximum in (kh,kw) scan order) as one byte
// per output element; backward is a deterministic gather over the <= ceil(k/s)^2 windows that
// cover an input pixel.  One thread = 8 channels (16-byte vectors), channels innermost.
// Also VGG's 2x2 / stride-2 VALID pool with the ReLU's derivative in its route bytes, and the standalone ReLU gate.
#include <cuda_bf16.h>

#include "common.cuh"

namespace rigl {

struct PoolGeom {
  int n, h, w, c, oh, ow, k, s, pad;
};

__global__ void __launch_bounds__(256)
k_maxpool_fwd(PoolGeom g, const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y,
              uint8_t* __restrict__ idx) {
  // grid = (column tiles, output rows, images), block = (8 channel vectors, 32 columns): no index
  // divisions in the kernel (they cost more than the window loads).
  const int V = g.c >> 3;
  const int ow = blockIdx.x * blockDim.y + threadIdx.y, oh = blockIdx.y, n = blockIdx.z;
  if (ow >= g.ow) return;
  const long long p = ((long long)n * g.oh + oh) * g.ow + ow;
  for (int v = threadIdx.x; v < V; v += blockDim.x) {
    float best[8];
    uint8_t arg[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) { best[e] = -INFINITY; arg[e] = 0; }
    for (int kh = 0; kh < g.k; ++kh) {
      const int hi = oh * g.s + kh - g.pad;
      if (hi < 0 || hi >= g.h) continue;
      for (int kw = 0; kw < g.k; ++kw) {
        const int wi = ow * g.s + kw - g.pad;
        if (wi < 0 || wi >= g.w) continue;
        const uint4 raw = *reinterpret_cast<const uint4*>(x + (((long long)n * g.h + hi) * g.w + wi) * g.c + 8 * v);
        const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&raw);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 f = __bfloat1622float2(h2[e]);
          if (f.x > best[2 * e]) { best[2 * e] = f.x; arg[2 * e] = (uint8_t)(kh * g.k + kw); }
          if (f.y > best[2 * e + 1]) { best[2 * e + 1] = f.y; arg[2 * e + 1] = (uint8_t)(kh * g.k + kw); }
        }
      }
    }
    uint4 o;
    __nv_bfloat162* oh2 = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
    for (int e = 0; e < 4; ++e) oh2[e] = __floats2bfloat162_rn(best[2 * e], best[2 * e + 1]);
    *reinterpret_cast<uint4*>(y + p * g.c + 8 * v) = o;
    uint2 a;
    a.x = arg[0] | (arg[1] << 8) | (arg[2] << 16) | ((uint32_t)arg[3] << 24);
    a.y = arg[4] | (arg[5] << 8) | (arg[6] << 16) | ((uint32_t)arg[7] << 24);
    *reinterpret_cast<uint2*>(idx + p * g.c + 8 * v) = a;
  }
}

__global__ void __launch_bounds__(256)
k_maxpool_bwd(PoolGeom g, const __nv_bfloat16* __restrict__ dy, const uint8_t* __restrict__ idx,
              __nv_bfloat16* __restrict__ dx) {
  const int V = g.c >> 3;
  const int wi = blockIdx.x * blockDim.y + threadIdx.y, hi = blockIdx.y, n = blockIdx.z;
  if (wi >= g.w) return;
  const long long q = ((long long)n * g.h + hi) * g.w + wi;
  // outputs oh with oh*s - pad <= hi <= oh*s - pad + k - 1
  const int oh_lo = max(0, (hi + g.pad - g.k + g.s) / g.s), oh_hi = min(g.oh - 1, (hi + g.pad) / g.s);
  const int ow_lo = max(0, (wi + g.pad - g.k + g.s) / g.s), ow_hi = min(g.ow - 1, (wi + g.pad) / g.s);
  for (int v = threadIdx.x; v < V; v += blockDim.x) {
    float acc[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] = 0.f;
    for (int oh = oh_lo; oh <= oh_hi; ++oh)
      for (int ow = ow_lo; ow <= ow_hi; ++ow) {
        const int rel = (hi - (oh * g.s - g.pad)) * g.k + (wi - (ow * g.s - g.pad));
        const long long p = ((long long)n * g.oh + oh) * g.ow + ow;
        const uint2 a = *reinterpret_cast<const uint2*>(idx + p * g.c + 8 * v);
        const uint4 raw = *reinterpret_cast<const uint4*>(dy + p * g.c + 8 * v);
        const __nv_bfloat16* d = reinterpret_cast<const __nv_bfloat16*>(&raw);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const uint32_t ai = ((e < 4 ? a.x : a.y) >> (8 * (e & 3))) & 0xFFu;
          if ((int)ai == rel) acc[e] += __bfloat162float(d[e]);
        }
      }
    uint4 o;
    __nv_bfloat162* o2 = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
    for (int e = 0; e < 4; ++e) o2[e] = __floats2bfloat162_rn(acc[2 * e], acc[2 * e + 1]);
    *reinterpret_cast<uint4*>(dx + q * g.c + 8 * v) = o;
  }
}

// The stem's case (3x3 window, stride 2, no leading pad, even extents): a 2x2 quad of input pixels is covered by the
// same four windows (oh-1|oh) x (ow-1|ow), nine (pixel, window) visits in all.  One thread = one quad x 8 channels:
// it loads the four outputs once (2.25 -> 1 window loads per input pixel) and writes the four pixels as two 32-byte
// runs.  Same accumulation order as the generic gather (oh ascending, then ow): bit-identical results.
__global__ void __launch_bounds__(256)
k_maxpool_bwd_3x3s2(PoolGeom g, const __nv_bfloat16* __restrict__ dy, const uint8_t* __restrict__ idx,
                    __nv_bfloat16* __restrict__ dx) {
  const int V = g.c >> 3;
  const int qw = blockIdx.x * blockDim.y + threadIdx.y, qh = blockIdx.y, n = blockIdx.z;
  if (qw >= (g.w >> 1)) return;
  for (int v = threadIdx.x; v < V; v += blockDim.x) {
    float acc[4][8];            // pixels (0,0) (0,1) (1,0) (1,1) of the quad
#pragma unroll
    for (int p = 0; p < 4; ++p)
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[p][e] = 0.f;
    uint2 a[4];
    uint4 d[4];
    bool ok[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {           // windows in the generic kernel's visiting order
      const int oh = qh - 1 + (j >> 1), ow = qw - 1 + (j & 1);
      ok[j] = oh >= 0 && ow >= 0 && oh < g.oh && ow < g.ow;
      a[j] = make_uint2(0xFFFFFFFFu, 0xFFFFFFFFu);
      d[j] = make_uint4(0u, 0u, 0u, 0u);
      if (ok[j]) {
        const long long p = (((long long)n * g.oh + oh) * g.ow + ow) * g.c + 8 * v;
        a[j] = *reinterpret_cast<const uint2*>(idx + p);
        d[j] = *reinterpret_cast<const uint4*>(dy + p);
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const __nv_bfloat16* dv = reinterpret_cast<const __nv_bfloat16*>(&d[j]);
      const int dh = 2 - 2 * (j >> 1), dw = 2 - 2 * (j & 1);   // window-relative position of pixel (0,0)
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int ai = (int)(((e < 4 ? a[j].x : a[j].y) >> (8 * (e & 3))) & 0xFFu);
        const float f = __bfloat162float(dv[e]);
#pragma unroll
        for (int p = 0; p < 4; ++p) {
          const int rh = dh + (p >> 1), rw = dw + (p & 1);
          if (rh < 3 && rw < 3 && ai == rh * 3 + rw) acc[p][e] += f;
        }
      }
    }
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      uint4 o;
      __nv_bfloat162* o2 = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
      for (int e = 0; e < 4; ++e) o2[e] = __floats2bfloat162_rn(acc[p][2 * e], acc[p][2 * e + 1]);
      const long long q = ((long long)n * g.h + 2 * qh + (p >> 1)) * g.w + 2 * qw + (p & 1);
      *reinterpret_cast<uint4*>(dx + q * g.c + 8 * v) = o;
    }
  }
}

// ---- VGG's 2x2 / stride-2 VALID max pool (layers.max_pool2d([2, 2]), vgg.py) over a ReLU output ----
// Forward: one thread = one output x 8 channels; it reads the four window pixels and stores the max and a route byte:
// the window-relative index (kh * 2 + kw) of the first maximum in scan order, or kNoRoute when that maximum is not
// > 0.  Backward: the windows are disjoint, so one thread writes its four input pixels directly (no gather);
// gradient goes only to a routed argmax.  A maximum that is not > 0 comes from a window the ReLU zeroed entirely, so
// the route byte also applies the ReLU's derivative: the producing conv receives the pre-activation gradient.
// Rows / columns past the last window (odd extents, VALID floor) get zero gradient.
constexpr uint8_t kNoRoute = 0xFF;

__global__ void __launch_bounds__(256)
k_maxpool2x2_relu_fwd(PoolGeom g, const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y,
                      uint8_t* __restrict__ idx) {
  const int V = g.c >> 3;
  const int ow = blockIdx.x * blockDim.y + threadIdx.y, oh = blockIdx.y, n = blockIdx.z;
  if (ow >= g.ow) return;
  const long long p = ((long long)n * g.oh + oh) * g.ow + ow;
  for (int v = threadIdx.x; v < V; v += blockDim.x) {
    uint4 raw[4];
#pragma unroll
    for (int j = 0; j < 4; ++j)
      raw[j] = *reinterpret_cast<const uint4*>(
          x + (((long long)n * g.h + 2 * oh + (j >> 1)) * g.w + 2 * ow + (j & 1)) * g.c + 8 * v);
    uint4 o;
    __nv_bfloat16* ob = reinterpret_cast<__nv_bfloat16*>(&o);
    uint32_t a[2] = {0u, 0u};
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      float best = __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(&raw[0])[e]);
      uint32_t arg = 0;
#pragma unroll
      for (int j = 1; j < 4; ++j) {
        const float f = __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(&raw[j])[e]);
        if (f > best) { best = f; arg = (uint32_t)j; }
      }
      ob[e] = __float2bfloat16_rn(best);                 // exact: best is one of the bf16 inputs
      a[e >> 2] |= (best > 0.f ? arg : (uint32_t)kNoRoute) << (8 * (e & 3));
    }
    *reinterpret_cast<uint4*>(y + p * g.c + 8 * v) = o;
    *reinterpret_cast<uint2*>(idx + p * g.c + 8 * v) = make_uint2(a[0], a[1]);
  }
}

// grid = (quad-column tiles, quad rows, images) over ceil(h/2) x ceil(w/2) quads
__global__ void __launch_bounds__(256)
k_maxpool2x2_relu_bwd(PoolGeom g, const __nv_bfloat16* __restrict__ dy, const uint8_t* __restrict__ idx,
                      __nv_bfloat16* __restrict__ dx) {
  const int V = g.c >> 3;
  const int qw = blockIdx.x * blockDim.y + threadIdx.y, qh = blockIdx.y, n = blockIdx.z;
  if (2 * qw >= g.w) return;
  const bool covered = qh < g.oh && qw < g.ow;
  for (int v = threadIdx.x; v < V; v += blockDim.x) {
    uint2 a = make_uint2(0xFFFFFFFFu, 0xFFFFFFFFu);
    uint4 d = make_uint4(0u, 0u, 0u, 0u);
    if (covered) {
      const long long p = (((long long)n * g.oh + qh) * g.ow + qw) * g.c + 8 * v;
      a = *reinterpret_cast<const uint2*>(idx + p);
      d = *reinterpret_cast<const uint4*>(dy + p);
    }
    const uint16_t* dv = reinterpret_cast<const uint16_t*>(&d);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int hi = 2 * qh + (j >> 1), wi = 2 * qw + (j & 1);
      if (hi >= g.h || wi >= g.w) continue;
      uint4 o;
      uint16_t* ov = reinterpret_cast<uint16_t*>(&o);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const uint32_t ai = ((e < 4 ? a.x : a.y) >> (8 * (e & 3))) & 0xFFu;
        ov[e] = ai == (uint32_t)j ? dv[e] : (uint16_t)0;
      }
      *reinterpret_cast<uint4*>(dx + (((long long)n * g.h + hi) * g.w + wi) * g.c + 8 * v) = o;
    }
  }
}

// out = x > 0 ? g : 0 over n bf16 elements (8 per thread); out may alias x or g.  With g == x it is the ReLU.
__global__ void __launch_bounds__(256)
k_relu_gate(const __nv_bfloat16* x, const __nv_bfloat16* gr, __nv_bfloat16* out, long long n8) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
    const uint4 xv = reinterpret_cast<const uint4*>(x)[i];
    const uint4 gv = reinterpret_cast<const uint4*>(gr)[i];
    const __nv_bfloat16* xb = reinterpret_cast<const __nv_bfloat16*>(&xv);
    const uint16_t* gb = reinterpret_cast<const uint16_t*>(&gv);
    uint4 o;
    uint16_t* ob = reinterpret_cast<uint16_t*>(&o);
#pragma unroll
    for (int e = 0; e < 8; ++e) ob[e] = __bfloat162float(xb[e]) > 0.f ? gb[e] : (uint16_t)0;
    reinterpret_cast<uint4*>(out)[i] = o;
  }
}

static int pool_geom(int n, int h, int w, int c, int k, int s, PoolGeom* g) {
  RIGL_REQUIRE(n > 0 && h > 0 && w > 0 && c > 0 && c % 8 == 0 && k > 0 && s > 0 && k * k <= 255,
               "maxpool: bad geometry (channels must be a multiple of 8)");
  g->n = n; g->h = h; g->w = w; g->c = c; g->k = k; g->s = s;
  g->oh = (h + s - 1) / s; g->ow = (w + s - 1) / s;                       // TF 'SAME'
  const int pad_total = max((g->oh - 1) * s + k - h, 0);
  g->pad = pad_total / 2;
  return RIGL_OK;
}

}  // namespace rigl

using namespace rigl;

extern "C" int rigl_maxpool_same_forward(const void* x, int n, int h, int w, int c, int ksize, int stride,
                                         void* y, uint8_t* argmax, void* stream) {
  PoolGeom g;
  int rc = pool_geom(n, h, w, c, ksize, stride, &g);
  if (rc != RIGL_OK) return rc;
  RIGL_REQUIRE(x && y && argmax, "rigl_maxpool_same_forward: null tensor");
  RIGL_REQUIRE(g.oh <= 65535 && n <= 65535, "rigl_maxpool_same_forward: extent too large");
  const dim3 block(8, 32), grid((unsigned)((g.ow + 31) / 32), (unsigned)g.oh, (unsigned)n);
  k_maxpool_fwd<<<grid, block, 0, (cudaStream_t)stream>>>(g, (const __nv_bfloat16*)x, (__nv_bfloat16*)y, argmax);
  RIGL_LAUNCH_CHECK("k_maxpool_fwd");
  return RIGL_OK;
}

extern "C" int rigl_maxpool_same_backward(const void* dy, const uint8_t* argmax, int n, int h, int w, int c,
                                          int ksize, int stride, void* dx, void* stream) {
  PoolGeom g;
  int rc = pool_geom(n, h, w, c, ksize, stride, &g);
  if (rc != RIGL_OK) return rc;
  RIGL_REQUIRE(dy && dx && argmax, "rigl_maxpool_same_backward: null tensor");
  RIGL_REQUIRE(g.h <= 65535 && n <= 65535, "rigl_maxpool_same_backward: extent too large");
  if (g.k == 3 && g.s == 2 && g.pad == 0 && (g.h & 1) == 0 && (g.w & 1) == 0) {
    const dim3 block(8, 32), grid((unsigned)((g.w / 2 + 31) / 32), (unsigned)(g.h / 2), (unsigned)n);
    k_maxpool_bwd_3x3s2<<<grid, block, 0, (cudaStream_t)stream>>>(g, (const __nv_bfloat16*)dy, argmax,
                                                                   (__nv_bfloat16*)dx);
    RIGL_LAUNCH_CHECK("k_maxpool_bwd_3x3s2");
    return RIGL_OK;
  }
  const dim3 block(8, 32), grid((unsigned)((g.w + 31) / 32), (unsigned)g.h, (unsigned)n);
  k_maxpool_bwd<<<grid, block, 0, (cudaStream_t)stream>>>(g, (const __nv_bfloat16*)dy, argmax, (__nv_bfloat16*)dx);
  RIGL_LAUNCH_CHECK("k_maxpool_bwd");
  return RIGL_OK;
}

extern "C" int rigl_maxpool2x2_relu_forward(const void* x, int n, int h, int w, int c, void* y, uint8_t* argmax,
                                            void* stream) {
  RIGL_REQUIRE(x && y && argmax, "rigl_maxpool2x2_relu_forward: null tensor");
  RIGL_REQUIRE(n > 0 && h >= 2 && w >= 2 && c > 0 && c % 8 == 0,
               "rigl_maxpool2x2_relu_forward: bad geometry (extents >= 2, channels a multiple of 8)");
  RIGL_REQUIRE(aligned16(x) && aligned16(y) && ((uintptr_t)argmax & 7) == 0,
               "rigl_maxpool2x2_relu_forward: x and y must be 16-byte, argmax 8-byte aligned");
  RIGL_REQUIRE(h / 2 <= 65535 && n <= 65535, "rigl_maxpool2x2_relu_forward: extent too large");
  const PoolGeom g = {n, h, w, c, h / 2, w / 2, 2, 2, 0};
  const dim3 block(8, 32), grid((unsigned)((g.ow + 31) / 32), (unsigned)g.oh, (unsigned)n);
  k_maxpool2x2_relu_fwd<<<grid, block, 0, (cudaStream_t)stream>>>(g, (const __nv_bfloat16*)x, (__nv_bfloat16*)y,
                                                                   argmax);
  RIGL_LAUNCH_CHECK("k_maxpool2x2_relu_fwd");
  return RIGL_OK;
}

extern "C" int rigl_maxpool2x2_relu_backward(const void* dy, const uint8_t* argmax, int n, int h, int w, int c,
                                             void* dx, void* stream) {
  RIGL_REQUIRE(dy && argmax && dx, "rigl_maxpool2x2_relu_backward: null tensor");
  RIGL_REQUIRE(n > 0 && h >= 2 && w >= 2 && c > 0 && c % 8 == 0,
               "rigl_maxpool2x2_relu_backward: bad geometry (extents >= 2, channels a multiple of 8)");
  RIGL_REQUIRE(aligned16(dy) && aligned16(dx) && ((uintptr_t)argmax & 7) == 0,
               "rigl_maxpool2x2_relu_backward: dy and dx must be 16-byte, argmax 8-byte aligned");
  RIGL_REQUIRE((h + 1) / 2 <= 65535 && n <= 65535, "rigl_maxpool2x2_relu_backward: extent too large");
  const PoolGeom g = {n, h, w, c, h / 2, w / 2, 2, 2, 0};
  const int qh = (h + 1) / 2, qw = (w + 1) / 2;
  const dim3 block(8, 32), grid((unsigned)((qw + 31) / 32), (unsigned)qh, (unsigned)n);
  k_maxpool2x2_relu_bwd<<<grid, block, 0, (cudaStream_t)stream>>>(g, (const __nv_bfloat16*)dy, argmax,
                                                                   (__nv_bfloat16*)dx);
  RIGL_LAUNCH_CHECK("k_maxpool2x2_relu_bwd");
  return RIGL_OK;
}

extern "C" int rigl_relu_gate(const void* x, const void* g, int64_t n, void* out, void* stream) {
  RIGL_REQUIRE(x && g && out, "rigl_relu_gate: null tensor");
  RIGL_REQUIRE(n > 0 && n % 8 == 0, "rigl_relu_gate: n = %lld is not a positive multiple of 8", (long long)n);
  RIGL_REQUIRE(aligned16(x) && aligned16(g) && aligned16(out), "rigl_relu_gate: tensors must be 16-byte aligned");
  const long long n8 = n / 8;
  long long blocks = (n8 + 255) / 256;
  if (blocks > kNumSmsHint * 16) blocks = kNumSmsHint * 16;
  k_relu_gate<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)x, (const __nv_bfloat16*)g,
                                                                  (__nv_bfloat16*)out, n8);
  RIGL_LAUNCH_CHECK("k_relu_gate");
  return RIGL_OK;
}
