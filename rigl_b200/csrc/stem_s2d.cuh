// Space-to-depth stem kernels (layers.STEM_S2D_PATH, default on; tests/test_conv_gpu.py::test_conv_stem_s2d_path).
// Design: DESIGN.md 3.2.
//
// The 7x7 / stride-2 / 3-channel stem without a patch matrix.  The zero-padded input is folded
// 2x2 -> channels ("space to depth"): xs[n, hs, ws, (dy*2+dx)*3 + c] = xpad[n, 2hs+dy, 2ws+dx, c],
// 16 bf16 = 32 bytes per folded pixel (slots 12..15 zero).  The conv becomes a 4x4 / stride-1
// conv over 16 channels (taps (th, tw), weights of the non-existent kh = 7 / kw = 7 zero), i.e.
// exactly ONE K = 16 wgmma per tap, and the halo trick of halo3x3.cuh applies with 32-byte rows:
// one halo tile of (R+3) folded rows x 128 columns (TMA, SWIZZLE_32B, OOB zero fill) feeds all 16
// taps; the A fragment of tap (th, tw) starts th*128 + tw rows down the tile and is loaded with
// ldmatrix at explicitly swizzled addresses.  An M tile is one output row (128 positions, 112 valid);
// the 32 KB weight operand stays resident.
//
// wgrad: for filter row th, D_th[tw*16 + k16][co] = sum_q xs_tile[q + th*128 + tw][k16] * dY[q][co] over the
// four horizontal taps tw = 0..3: M = 64, one wgmma per (th, 16 positions), A = the shifted tile read transposed
// (ldmatrix.trans), B = the dY tile (MN-major, SWIZZLE_128B, padding columns zero-filled by TMA).  Per-CTA fp32
// partials [th][tw*16 + k16][co] (rows 64..127 of each th block unused), then k_stem_s2d_reduce scatters them
// into the dense HWIO gradient in CTA order (deterministic).
//
// Output channels come in groups of 64 (blockIdx.y): a CTA of group j holds the weight rows 64j .. 64j+63 and
// writes / reads the output-gradient channels of that box; a ragged last group is zero-filled by the weight and
// dY loads and clipped by the output store.  Every group runs the grid and strip order of a 64-channel launch, so
// each group's output and gradient are those of a separate launch on its weight slice.
//
// Included by igemm_tc.cu inside namespace rigl.
#pragma once

struct S2dParams {
  int H, W;                     // output extents (conv output = in/2)
  int NB;
  int HS, WS;                   // folded input extents: (in + 2*pad) / 2
  int R;                        // output rows per strip (= M tiles per strip)
  int nbuf;
  int strips_per_image, total_strips;
  int N;                        // output channels (<= 256)
  int groups;                   // 64-channel groups: gridDim.y
  uint32_t a_buf_bytes;         // halo tile incl. slack rows, multiple of 1024
  uint32_t a_tx_bytes;
  float* wgrad_out;             // wgrad: [gridDim.x][groups][4][128][64] fp32
};

constexpr int kS2dWp = 128;                               // halo pitch (positions per M tile)
constexpr uint32_t kS2dBTapBytes = 64 * 16 * 2;           // one tap of the weight operand: 64 rows x 32 B

// ---- input fold: x [N,H,W,cin<=3] (pitch x_pitch) -> xs [N,HS,WS,16] ----
__global__ void __launch_bounds__(256)
k_stem_s2d_fold(ConvGeom g, int hs, int ws, const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ xs) {
  const long long total = (long long)g.batch * hs * ws;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int wx = (int)(i % ws), hy = (int)((i / ws) % hs), n = (int)(i / ((long long)ws * hs));
    __align__(16) __nv_bfloat16 v[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) v[k] = __float2bfloat16(0.f);
#pragma unroll
    for (int dy = 0; dy < 2; ++dy)
#pragma unroll
      for (int dx = 0; dx < 2; ++dx) {
        const int hi = 2 * hy + dy - g.pad, wi = 2 * wx + dx - g.pad;
        if (hi >= 0 && hi < g.in_h && wi >= 0 && wi < g.in_w) {
          const __nv_bfloat16* src = x + (((long long)n * g.in_h + hi) * g.in_w + wi) * g.x_pitch;
          for (int c = 0; c < g.cin; ++c) v[(dy * 2 + dx) * 3 + c] = src[c];
        }
      }
    uint4* dst = reinterpret_cast<uint4*>(xs + i * 16);
    dst[0] = reinterpret_cast<const uint4*>(v)[0];
    dst[1] = reinterpret_cast<const uint4*>(v)[1];
  }
}

// ---- weights: fp32 HWIO [7][7][cin][cout] + bitmap -> bf16 [16 taps][cout][16] (mask fused) ----
__global__ void __launch_bounds__(256)
k_stem_s2d_pack(ConvGeom g, const float* __restrict__ w, const uint32_t* __restrict__ bits,
                __nv_bfloat16* __restrict__ out) {
  const int total = 16 * g.cout * 16;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int k16 = i % 16, co = (i / 16) % g.cout, tap = i / (16 * g.cout);
  const int th = tap / 4, tw = tap % 4, q = k16 / 3, c = k16 % 3;
  const int kh = 2 * th + (q >> 1), kw = 2 * tw + (q & 1);
  float v = 0.f;
  if (k16 < 12 && c < g.cin && kh < g.ksize && kw < g.ksize) {
    const long long flat = (((long long)kh * g.ksize + kw) * g.cin + c) * g.cout + co;
    if ((bits[flat >> 5] >> (flat & 31)) & 1u) v = w[flat];
  }
  out[i] = __float2bfloat16(v);
}

// ---- forward ----
__global__ void __launch_bounds__(kThreads, 1)
k_stem_s2d_fprop(const __grid_constant__ CUtensorMap amap, const __grid_constant__ CUtensorMap bmap,
                 const __grid_constant__ CUtensorMap omap, const S2dParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  constexpr uint32_t kSlab = 128 * 64 * 2;
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t b_base = smem_base;                                   // 16 taps x 2 KB
  const uint32_t a_base = b_base + 16 * kS2dBTapBytes;
  const uint32_t out_base = a_base + p.nbuf * p.a_buf_bytes;
  const uint32_t bar_base = out_base + 2 * kSlab;
  const uint32_t b_full = bar_base;
  auto a_full = [&](int b) { return bar_base + 8u * (1 + b); };
  auto a_empty = [&](int b) { return bar_base + 8u * (5 + b); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    prefetch_tmap(&amap); prefetch_tmap(&bmap); prefetch_tmap(&omap);
    mbar_init(b_full, 1);
    for (int b = 0; b < p.nbuf; ++b) { mbar_init(a_full(b), 1); mbar_init(a_empty(b), kConsumerWarps); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 0) {
    if (elect_one()) {
      mbar_arrive_expect_tx(b_full, 16 * kS2dBTapBytes);
      for (int t = 0; t < 16; ++t) tma_load_3d(b_base + t * kS2dBTapBytes, &bmap, b_full, 0, 64 * blockIdx.y, t);
      int buf = 0; uint32_t phase = 0;
      for (int strip = blockIdx.x; strip < p.total_strips; strip += gridDim.x) {
        const int n = strip / p.strips_per_image, h0 = (strip % p.strips_per_image) * p.R;
        mbar_wait(a_empty(buf), phase ^ 1u);
        mbar_arrive_expect_tx(a_full(buf), p.a_tx_bytes);
        tma_load_4d(a_base + buf * p.a_buf_bytes, &amap, a_full(buf), 0, 0, h0, n);   // folded rows h0 .. h0+R+2
        if (++buf == p.nbuf) { buf = 0; phase ^= 1u; }
      }
    }
    __syncwarp();
  } else if (warp >= kConsumerWarp0) {
    const int cw = warp - kConsumerWarp0;
    const int wg = cw >> 2;
    const int row = 64 * wg + 16 * (cw & 3) + (lane >> 2);
    const int lrow = 64 * wg + 16 * (cw & 3) + (lane & 7) + 8 * ((lane >> 3) & 1);
    const uint32_t lk = (uint32_t)(lane >> 4) * 16u;
    const bool issuer = (cw == 0 && lane == 0);
    const uint64_t b_desc0 = make_smem_desc(b_base, 16, 256, kSwz32);
    mbar_wait(b_full, 0);
    int buf = 0; uint32_t phase = 0;
    uint32_t slab_ctr = 0;
    for (int strip = blockIdx.x; strip < p.total_strips; strip += gridDim.x) {
      const int n = strip / p.strips_per_image, h0 = (strip % p.strips_per_image) * p.R;
      mbar_wait(a_full(buf), phase);
      const uint32_t a_tile = a_base + buf * p.a_buf_bytes;
      for (int t = 0; t < p.R; ++t) {                        // M tile t = output row h0 + t
        float acc[32];
        zero_acc(acc);
        uint32_t a[2][4];
#pragma unroll
        for (int tap = 0; tap < 16; ++tap) {                 // rows of 32 B
          const int r = (t + (tap >> 2)) * kS2dWp + (tap & 3) + lrow;
          ldmatrix_x4(a[tap & 1], swz32(a_tile + (uint32_t)r * 32u + lk));
          fence_regs(acc);
          wgmma_fence();
          Wgmma<64>::rs<0>(acc, a[tap & 1], b_desc0 + (uint64_t)(tap * (kS2dBTapBytes >> 4)));
          wgmma_commit();
          wgmma_wait<1>();
          if (tap > 0) keep_frag(a[(tap + 1) & 1]);
        }
        wgmma_wait<0>();
        fence_regs(acc);
        keep_frag(a[1]);
        const uint32_t slab = out_base + (slab_ctr & 1u) * kSlab;
        if (issuer) tma_store_wait_read<1>();
        named_bar_sync(1, kConsumerThreads);
        stage_slab<0>(acc, slab, row, true, true, lane);     // columns >= W and rows >= H are clipped by the store
        fence_proxy_async_smem();
        named_bar_sync(1, kConsumerThreads);
        if (issuer) {
          tma_store_4d(&omap, slab, 64 * blockIdx.y, 0, h0 + t, n);
          tma_store_commit();
        }
        ++slab_ctr;
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(a_empty(buf));
      if (++buf == p.nbuf) { buf = 0; phase ^= 1u; }
    }
    if (issuer) tma_store_wait_all();
  }
}

// ---- wgrad ----
// Consumer warpgroup wg accumulates filter rows th = 2wg, 2wg + 1; warp w of it owns the rows tw = w of both.
__global__ void __launch_bounds__(kThreads, 1)
k_stem_s2d_wgrad(const __grid_constant__ CUtensorMap xmap, const __grid_constant__ CUtensorMap dymap,
                 const S2dParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t dy_bytes = (uint32_t)(p.R * kS2dWp) * 128u;
  const uint32_t stage_bytes = p.a_buf_bytes + dy_bytes;               // [x halo | dy]
  const uint32_t bar_base = smem_base + p.nbuf * stage_bytes;
  auto full_bar = [&](int b) { return bar_base + 8u * b; };
  auto empty_bar = [&](int b) { return bar_base + 8u * (4 + b); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    prefetch_tmap(&xmap); prefetch_tmap(&dymap);
    for (int b = 0; b < p.nbuf; ++b) { mbar_init(full_bar(b), 1); mbar_init(empty_bar(b), kConsumerWarps); }
    fence_barrier_init();
  }
  {   // slack rows behind each halo tile are read against zero dY columns: they must be finite
    const uint32_t slack = p.a_buf_bytes - p.a_tx_bytes;
    for (int b = 0; b < p.nbuf; ++b)
      for (uint32_t i = threadIdx.x * 16u; i < slack; i += kThreads * 16u)
        asm volatile("st.shared.v4.b32 [%0], {%1, %1, %1, %1};" ::"r"(smem_base + b * stage_bytes + p.a_tx_bytes + i), "r"(0u)
                     : "memory");
    fence_proxy_async_smem();
  }
  __syncthreads();

  if (warp == 0) {
    if (elect_one()) {
      int buf = 0; uint32_t phase = 0;
      for (int strip = blockIdx.x; strip < p.total_strips; strip += gridDim.x) {
        const int n = strip / p.strips_per_image, h0 = (strip % p.strips_per_image) * p.R;
        mbar_wait(empty_bar(buf), phase ^ 1u);
        mbar_arrive_expect_tx(full_bar(buf), p.a_tx_bytes + dy_bytes);
        const uint32_t x_dst = smem_base + buf * stage_bytes;
        tma_load_4d(x_dst, &xmap, full_bar(buf), 0, 0, h0, n);
        tma_load_4d(x_dst + p.a_buf_bytes, &dymap, full_bar(buf), 64 * blockIdx.y, 0, h0, n);
        if (++buf == p.nbuf) { buf = 0; phase ^= 1u; }
      }
    }
    __syncwarp();
  } else if (warp >= kConsumerWarp0) {
    const int cw = warp - kConsumerWarp0;
    const int wg = cw >> 2, tw = cw & 3;
    // ldmatrix.trans: lane supplies position (K) row 8 * (lane >> 4) + (lane & 7) of matrix lane / 8, whose 8
    // folded channels are the 16-byte half (lane >> 3) & 1 of the 32-byte row.
    const uint32_t lpos = (uint32_t)(8 * (lane >> 4) + (lane & 7));
    const uint32_t lhalf = (uint32_t)((lane >> 3) & 1) * 16u;
    float acc[2][32];
    zero_acc(acc[0]); zero_acc(acc[1]);
    uint32_t a[2][4];
    int buf = 0; uint32_t phase = 0;
    const int ksteps = p.R * kS2dWp / 16;
    for (int strip = blockIdx.x; strip < p.total_strips; strip += gridDim.x) {
      mbar_wait(full_bar(buf), phase);
      const uint32_t x_src = smem_base + buf * stage_bytes;
      const uint64_t db0 = make_smem_desc(x_src + p.a_buf_bytes, 8192, 1024);     // dY: 128-byte rows
#pragma unroll 1
      for (int k = 0; k < ksteps; ++k) {                   // 16 positions: +512 B of x rows, +2048 B of dY rows
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int th = 2 * wg + i;
          const uint32_t r = (uint32_t)(16 * k + th * kS2dWp + tw) + lpos;
          ldmatrix_x4_trans(a[i], swz32(x_src + r * 32u + lhalf));
          fence_regs(acc[i]);
          wgmma_fence();
          Wgmma<64>::rs<1>(acc[i], a[i], db0 + (uint64_t)(128 * k));
          wgmma_commit();
          wgmma_wait<1>();                                 // the MMA that last read a[i ^ 1] has retired
          keep_frag(a[i ^ 1]);
        }
      }
      wgmma_wait<0>();
      fence_regs(acc[0]); fence_regs(acc[1]);
      keep_frag(a[0]); keep_frag(a[1]);
      __syncwarp();
      if (lane == 0) mbar_arrive(empty_bar(buf));
      if (++buf == p.nbuf) { buf = 0; phase ^= 1u; }
    }
    float* part = p.wgrad_out + ((size_t)blockIdx.x * p.groups + blockIdx.y) * 4 * 128 * 64;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int th = 2 * wg + i;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float* dst_row = part + ((size_t)th * 128 + tw * 16 + (lane >> 2) + 8 * h) * 64;
#pragma unroll
        for (int jc = 0; jc < 8; ++jc)
          *reinterpret_cast<float2*>(dst_row + 8 * jc + 2 * (lane & 3)) =
              make_float2(acc[i][4 * jc + 2 * h], acc[i][4 * jc + 2 * h + 1]);
      }
    }
  }
}

// dw[kh][kw][c][co] = beta * dw + sum over CTAs of partial[cta][co/64][kh/2][(kw/2)*16 + ((kh&1)*2 + (kw&1))*3 + c][co%64]
__global__ void __launch_bounds__(256)
k_stem_s2d_reduce(ConvGeom g, const float* __restrict__ part, int nparts, int groups, float* __restrict__ dw,
                  float beta) {
  const int total = g.ksize * g.ksize * g.cin * g.cout;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int co = i % g.cout, c = (i / g.cout) % g.cin, kw = (i / (g.cout * g.cin)) % g.ksize, kh = i / (g.cout * g.cin * g.ksize);
  const int th = kh >> 1, row = (kw >> 1) * 16 + ((kh & 1) * 2 + (kw & 1)) * 3 + c;
  const float* src = part + (((size_t)(co >> 6) * 4 + th) * 128 + row) * 64 + (co & 63);
  const size_t cta_stride = (size_t)groups * 4 * 128 * 64;
  float a = beta != 0.f ? beta * dw[i] : 0.f;
  for (int s = 0; s < nparts; ++s) a += src[(size_t)s * cta_stride];
  dw[i] = a;
}

// ---------------------------------------------------------------------------- host side
static bool s2d_geom(const ConvGeom& g, S2dParams* p, bool wgrad) {
  if (g.ksize != 7 || g.stride != 2 || g.pad != 3 || g.cin > 3 || g.cin < 1) return false;
  if ((g.in_h & 1) || (g.in_w & 1) || g.cout > 256 || (g.cout % 8)) return false;
  if (g.out_h != g.in_h / 2 || g.out_w != g.in_w / 2 || g.out_w + 3 > kS2dWp) return false;
  p->H = g.out_h; p->W = g.out_w; p->NB = g.batch;
  p->HS = (g.in_h + 2 * g.pad) / 2; p->WS = (g.in_w + 2 * g.pad) / 2;
  p->R = wgrad ? 4 : 8;
  p->nbuf = wgrad ? 2 : 3;
  if (p->R > g.out_h) p->R = g.out_h;
  p->strips_per_image = (g.out_h + p->R - 1) / p->R;
  p->total_strips = p->strips_per_image * g.batch;
  p->N = g.cout;
  p->groups = (g.cout + 63) / 64;
  p->a_tx_bytes = (uint32_t)((p->R + 3) * kS2dWp) * 32u;
  p->a_buf_bytes = (uint32_t)(((size_t)((p->R + 3) * kS2dWp + 8) * 32 + 1023) / 1024 * 1024);
  p->wgrad_out = nullptr;
  return true;
}

bool s2d_supported(const ConvGeom& g) {
  S2dParams p;
  return s2d_geom(g, &p, false);
}
size_t s2d_folded_bytes(const ConvGeom& g) {
  S2dParams p;
  if (!s2d_geom(g, &p, false)) return 0;
  return (size_t)g.batch * p.HS * p.WS * 32;
}
size_t s2d_packed_bytes(const ConvGeom& g) { return (size_t)16 * g.cout * 32; }
static int s2d_wgrad_grid(const S2dParams& p) {
  ensure_driver();
  const int sms = g_num_sms > 0 ? g_num_sms : kNumSmsHint;
  return p.total_strips < sms ? p.total_strips : sms;
}
size_t s2d_workspace_bytes(const ConvGeom& g) {
  S2dParams p;
  if (!s2d_geom(g, &p, true)) return 0;
  return (size_t)s2d_wgrad_grid(p) * p.groups * 4 * 128 * 64 * sizeof(float) + 256;
}

int s2d_fold(const ConvGeom& g, const void* x, void* xs, cudaStream_t s) {
  S2dParams p;
  if (!s2d_geom(g, &p, false)) { set_error("rigl_stem_s2d: unsupported geometry"); return RIGL_ERR_UNSUPPORTED; }
  k_stem_s2d_fold<<<kNumSmsHint * 16, 256, 0, s>>>(g, p.HS, p.WS, (const __nv_bfloat16*)x, (__nv_bfloat16*)xs);
  RIGL_LAUNCH_CHECK("k_stem_s2d_fold");
  return RIGL_OK;
}

int s2d_pack(const ConvGeom& g, const float* w, const uint32_t* bits, void* packed, cudaStream_t s) {
  const int total = 16 * g.cout * 16;
  k_stem_s2d_pack<<<(total + 255) / 256, 256, 0, s>>>(g, w, bits, (__nv_bfloat16*)packed);
  RIGL_LAUNCH_CHECK("k_stem_s2d_pack");
  return RIGL_OK;
}

// folded-input view (16, WS, HS, N) with 32-byte rows
static int s2d_x_map(CUtensorMap* out, const void* xs, const S2dParams& p, int box_rows) {
  const uint64_t dims[4] = {16, (uint64_t)p.WS, (uint64_t)p.HS, (uint64_t)p.NB};
  const uint64_t strides[3] = {32, (uint64_t)p.WS * 32, (uint64_t)p.HS * p.WS * 32};
  const uint32_t box[4] = {16, (uint32_t)kS2dWp, (uint32_t)box_rows, 1};
  return make_tmap_swz(out, xs, 4, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_32B);
}

int s2d_fprop(const ConvGeom& g, const void* xs, const void* packed, void* y, cudaStream_t s) {
  int rc = ensure_driver();
  if (rc != RIGL_OK) return rc;
  S2dParams p;
  if (!s2d_geom(g, &p, false)) { set_error("rigl_stem_s2d_fprop: unsupported geometry"); return RIGL_ERR_UNSUPPORTED; }
  CUtensorMap amap, bmap, omap;
  rc = s2d_x_map(&amap, xs, p, p.R + 3);
  if (rc != RIGL_OK) return rc;
  const uint64_t bdims[3] = {16, (uint64_t)g.cout, 16};
  const uint64_t bstr[2] = {32, (uint64_t)g.cout * 32};
  const uint32_t bbox[3] = {16, 64, 1};
  rc = make_tmap_swz(&bmap, packed, 3, bdims, bstr, bbox, CU_TENSOR_MAP_SWIZZLE_32B);
  if (rc != RIGL_OK) return rc;
  const uint32_t obox[4] = {64, (uint32_t)kS2dWp, 1, 1};
  rc = make_act_map(&omap, y, g.batch, g.out_h, g.out_w, g.cout, g.cout, 1, 0, 0, obox);
  if (rc != RIGL_OK) return rc;
  const size_t smem = 16 * kS2dBTapBytes + p.nbuf * (size_t)p.a_buf_bytes + 2 * (128 * 64 * 2) + 1024 + 256;
  RIGL_CUDA(smem_limit<k_stem_s2d_fprop>(smem));
  const int sms = g_num_sms > 0 ? g_num_sms : kNumSmsHint;
  const dim3 grid(p.total_strips < sms ? p.total_strips : sms, p.groups);
  k_stem_s2d_fprop<<<grid, kThreads, smem, s>>>(amap, bmap, omap, p);
  RIGL_LAUNCH_CHECK("k_stem_s2d_fprop");
  return RIGL_OK;
}

int s2d_wgrad(const ConvGeom& g, const void* xs, const void* dy, float* dw, float beta, void* ws, size_t ws_bytes,
              cudaStream_t s) {
  int rc = ensure_driver();
  if (rc != RIGL_OK) return rc;
  S2dParams p;
  if (!s2d_geom(g, &p, true)) { set_error("rigl_stem_s2d_wgrad: unsupported geometry"); return RIGL_ERR_UNSUPPORTED; }
  const int grid = s2d_wgrad_grid(p);
  const size_t need = (size_t)grid * p.groups * 4 * 128 * 64 * sizeof(float);
  if (ws == nullptr || ws_bytes < need + 256) {
    set_error("rigl_stem_s2d_wgrad: workspace %zu < required %zu", ws_bytes, need + 256);
    return RIGL_ERR_WORKSPACE;
  }
  p.wgrad_out = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(ws) + 255) & ~(uintptr_t)255);
  CUtensorMap xmap, dymap;
  rc = s2d_x_map(&xmap, xs, p, p.R + 3);
  if (rc != RIGL_OK) return rc;
  const uint32_t dbox[4] = {64, (uint32_t)kS2dWp, (uint32_t)p.R, 1};
  rc = make_act_map(&dymap, dy, g.batch, g.out_h, g.out_w, g.cout, g.cout, 1, 0, 0, dbox);
  if (rc != RIGL_OK) return rc;
  const size_t smem = p.nbuf * ((size_t)p.a_buf_bytes + (size_t)p.R * kS2dWp * 128) + 1024 + 256;
  RIGL_CUDA(smem_limit<k_stem_s2d_wgrad>(smem));
  k_stem_s2d_wgrad<<<dim3(grid, p.groups), kThreads, smem, s>>>(xmap, dymap, p);
  RIGL_LAUNCH_CHECK("k_stem_s2d_wgrad");
  const int total = g.ksize * g.ksize * g.cin * g.cout;
  k_stem_s2d_reduce<<<(total + 255) / 256, 256, 0, s>>>(g, p.wgrad_out, grid, p.groups, dw, beta);
  RIGL_LAUNCH_CHECK("k_stem_s2d_reduce");
  return RIGL_OK;
}
