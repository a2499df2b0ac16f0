// 3x3 / stride 1 / pad 1 convolutions with at most 64 reduction channels ("halo" kernels).
//
// The generic implicit-GEMM kernels fetch one shifted TMA box per filter tap, so a 3x3 layer
// reads its input NINE times from L2; at 64 channels there is so little math per byte that the
// chip-wide L2 -> SM bandwidth is what bounds them.
// Here a CTA loads ONE halo tile -- (R+2) image rows, each padded to a power-of-two pitch Wp
// >= W+2 by TMA out-of-bounds zero fill -- and feeds all nine taps from it: the A operand of tap
// (dh, dw) simply starts (dh+1)*Wp + (dw+1) rows (128 B each) further down the tile.  Such a start
// is not aligned to the 1024-byte swizzle period, so the A fragments are loaded with ldmatrix at
// explicitly swizzled addresses (the TMA writes SWIZZLE_128B as a function of the absolute
// shared-memory address) and fed to the register-A form of wgmma; the B operands (resident
// weights, the dY tile) stay on aligned shared-memory descriptors.
//
//   position q = r*Wp + c   (r = row inside the strip, c = column, c >= W is padding)
//   fprop/dgrad: D[q, n]   = sum_tap sum_k  X[q + off(tap), k] * Wt[tap][n, k]     (K-major A)
//   wgrad:       D[tap][ci, co] = sum_q X[q + off(tap), ci] * dY[q, co]            (A = X^T via ldmatrix.trans)
// Padding columns of the OUTPUT are clipped by the TMA store (fprop/dgrad) or multiply dY zeros
// (wgrad: the dY tile is loaded with the same pitch, its padding columns zero-filled).
//
// Included by igemm_tc.cu (uses its tensor-map helpers).
#pragma once
// (textually included inside namespace rigl)

struct HaloParams {
  int W, H, NB;                 // image extents (input == output)
  int Wp;                       // halo row pitch in pixels: power of two, W + 2 <= Wp <= 128
  int R;                        // output rows per strip (multiple of 128 / Wp)
  int T;                        // 128-position M tiles per strip (R * Wp / 128)
  int nbuf;                     // halo tiles in flight (2..4)
  int strips_per_image, total_strips;
  int N;                        // fprop/dgrad: output channels.  wgrad: co
  int ci;                       // wgrad: input channels (<= 64)
  int row_off[9];               // halo row offset of each tap: (dh+1)*Wp + (dw+1)
  uint32_t a_buf_bytes;         // halo tile incl. slack rows, multiple of 1024
  uint32_t a_tx_bytes;          // bytes the halo TMA box delivers
  float* wgrad_out;             // wgrad: [gridDim.x][9][ci][N] fp32 partials
};

constexpr uint32_t kHaloBTapBytes = 64 * 64 * 2;        // one tap of the resident weight tile: 8 KB
constexpr uint32_t kHaloSlabBytes = 128 * 64 * 2;       // output staging slab: 16 KB
// wgrad: three consumer warpgroups, one per filter row, and no separate producer warpgroup (thread 0 issues the
// loads): at 384 threads a thread may hold 168 registers, room for the 96 accumulator registers of a filter row
// plus two steps of A fragments in flight without spilling or serialising the wgmma stream.
constexpr int kHaloWgradThreads = 384;

// The register-A fragments of an in-flight wgmma must keep their registers until the MMA has read them:
// `keep_frag` after the wait that retires the MMA keeps the values (and so their registers) live up to it.
__device__ __forceinline__ void keep_frag(const uint32_t (&a)[4]) {
  asm volatile("" ::"r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]) : "memory");
}

// ----------------------------------------------------------------------------
// fprop / dgrad: weights of this CTA's 64-channel N tile stay resident in shared memory.
// grid = (CTAs over strips, N tiles).  warp 0: TMA; warpgroups 1-2: MMA + epilogue, 64 positions of each
// 128-position M tile each.  kRelu: the fprop stores bf16(relu(D)) (stage_slab_relu).
// ----------------------------------------------------------------------------
template <bool kRelu>
__device__ __forceinline__ void halo_kmajor_body(const CUtensorMap& amap, const CUtensorMap& bmap,
                                                 const CUtensorMap& omap, const HaloParams& p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t b_base = smem_base;                                   // 9 taps x 8 KB
  const uint32_t a_base = b_base + 9 * kHaloBTapBytes;                 // nbuf halo tiles
  const uint32_t out_base = a_base + p.nbuf * p.a_buf_bytes;           // 2 staging slabs
  const uint32_t bar_base = out_base + 2 * kHaloSlabBytes;
  const uint32_t b_full = bar_base;
  auto a_full = [&](int b) { return bar_base + 8u * (1 + b); };
  auto a_empty = [&](int b) { return bar_base + 8u * (5 + b); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_tile = blockIdx.y;
  if (threadIdx.x == 0) {
    prefetch_tmap(&amap); prefetch_tmap(&bmap); prefetch_tmap(&omap);
    mbar_init(b_full, 1);
    for (int b = 0; b < p.nbuf; ++b) { mbar_init(a_full(b), 1); mbar_init(a_empty(b), kConsumerWarps); }
    fence_barrier_init();
  }
  __syncthreads();
  const int rt = 128 / p.Wp;                              // image rows per M tile

  if (warp == 0) {
    if (lane == 0) {
      mbar_arrive_expect_tx(b_full, 9 * kHaloBTapBytes);
      for (int t = 0; t < 9; ++t) tma_load_3d(b_base + t * kHaloBTapBytes, &bmap, b_full, 0, n_tile * 64, t);
      int buf = 0; uint32_t phase = 0;
      for (int strip = blockIdx.x; strip < p.total_strips; strip += gridDim.x) {
        const int n = strip / p.strips_per_image, h0 = (strip % p.strips_per_image) * p.R;
        mbar_wait(a_empty(buf), phase ^ 1u);
        mbar_arrive_expect_tx(a_full(buf), p.a_tx_bytes);
        tma_load_4d(a_base + buf * p.a_buf_bytes, &amap, a_full(buf), 0, -1, h0 - 1, n);
        if (++buf == p.nbuf) { buf = 0; phase ^= 1u; }
      }
    }
  } else if (warp >= kConsumerWarp0) {
    const int cw = warp - kConsumerWarp0;
    const int wg = cw >> 2;
    const int row = 64 * wg + 16 * (cw & 3) + (lane >> 2);             // accumulator rows row, row + 8
    // ldmatrix: lane supplies position lrow of matrix lane / 8 (rows +8 for matrices 1 and 3, K +8 for 2 and 3)
    const int lrow = 64 * wg + 16 * (cw & 3) + (lane & 7) + 8 * ((lane >> 3) & 1);
    const uint32_t lk = (uint32_t)(lane >> 4) * 16u;
    const bool issuer = (cw == 0 && lane == 0);
    const uint64_t b_desc0 = make_smem_desc(b_base, 16, 1024);
    mbar_wait(b_full, 0);
    int buf = 0; uint32_t phase = 0;
    uint32_t slab_ctr = 0;
    for (int strip = blockIdx.x; strip < p.total_strips; strip += gridDim.x) {
      const int n = strip / p.strips_per_image, h0 = (strip % p.strips_per_image) * p.R;
      mbar_wait(a_full(buf), phase);
      const uint32_t a_tile = a_base + buf * p.a_buf_bytes;
      for (int t = 0; t < p.T; ++t) {
        float acc[32];
        zero_acc(acc);
        uint32_t a[2][4][4];
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
          const uint32_t src = a_tile + (uint32_t)(t * 128 + lrow + p.row_off[tap]) * 128u + lk;
#pragma unroll
          for (int k = 0; k < 4; ++k) ldmatrix_x4(a[tap & 1][k], swz128(src + 32u * k));
          fence_regs(acc);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < 4; ++k)                     // descriptor start addresses are in 16-byte units
            Wgmma<64>::rs<0>(acc, a[tap & 1][k], b_desc0 + (uint64_t)(tap * (kHaloBTapBytes >> 4) + 2 * k));
          wgmma_commit();
          wgmma_wait<1>();                                // the previous tap's fragments may be overwritten
          if (tap > 0) {
#pragma unroll
            for (int k = 0; k < 4; ++k) keep_frag(a[(tap + 1) & 1][k]);
          }
        }
        wgmma_wait<0>();
        fence_regs(acc);
#pragma unroll
        for (int k = 0; k < 4; ++k) keep_frag(a[0][k]);
        const uint32_t slab = out_base + (slab_ctr & 1u) * kHaloSlabBytes;
        if (issuer) tma_store_wait_read<1>();
        named_bar_sync(1, kConsumerThreads);
        if (kRelu) stage_slab_relu<0, false>(acc, slab, row, true, true, lane);
        else stage_slab<0>(acc, slab, row, true, true, lane);   // columns >= W and rows >= H are clipped by the store
        fence_proxy_async_smem();
        named_bar_sync(1, kConsumerThreads);
        if (issuer) {
          tma_store_4d(&omap, slab, n_tile * 64, 0, h0 + t * rt, n);
          tma_store_commit();
        }
        ++slab_ctr;
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(a_empty(buf));           // every MMA of this warp that read the tile has retired
      if (++buf == p.nbuf) { buf = 0; phase ^= 1u; }
    }
    if (issuer) tma_store_wait_all();
  }
}

__global__ void __launch_bounds__(kThreads, 1)
k_halo3x3_kmajor(const __grid_constant__ CUtensorMap amap, const __grid_constant__ CUtensorMap bmap,
                 const __grid_constant__ CUtensorMap omap, const HaloParams p) {
  halo_kmajor_body<false>(amap, bmap, omap, p);
}

__global__ void __launch_bounds__(kThreads, 1)
k_halo3x3_kmajor_relu(const __grid_constant__ CUtensorMap amap, const __grid_constant__ CUtensorMap bmap,
                      const __grid_constant__ CUtensorMap omap, const HaloParams p) {
  halo_kmajor_body<true>(amap, bmap, omap, p);
}

// ----------------------------------------------------------------------------
// wgrad: every CTA accumulates all nine taps over its strips in registers -- consumer warpgroup kh holds the three 64 x 64 accumulators of filter row kh -- then writes one fp32 partial [9][ci][co]; k_splitk_reduce
// sums the partials in CTA order (deterministic).
// ----------------------------------------------------------------------------
__global__ void __launch_bounds__(kHaloWgradThreads, 1)
k_halo3x3_wgrad(const __grid_constant__ CUtensorMap xmap, const __grid_constant__ CUtensorMap dymap,
                const HaloParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  constexpr int kWarps = 12;                                           // consumer warps
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t dy_bytes = (uint32_t)(p.R * p.Wp) * 128u;
  const uint32_t stage_bytes = p.a_buf_bytes + dy_bytes;               // [x halo | dy]
  const uint32_t bar_base = smem_base + p.nbuf * stage_bytes;
  auto full_bar = [&](int b) { return bar_base + 8u * b; };
  auto empty_bar = [&](int b) { return bar_base + 8u * (4 + b); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    prefetch_tmap(&xmap); prefetch_tmap(&dymap);
    for (int b = 0; b < p.nbuf; ++b) { mbar_init(full_bar(b), 1); mbar_init(empty_bar(b), kWarps); }
    fence_barrier_init();
  }
  // The slack rows behind each halo tile are read (against zero dY columns): they must be finite.
  {
    const uint32_t halo_rows_bytes = p.a_tx_bytes;
    const uint32_t slack = p.a_buf_bytes - halo_rows_bytes;
    for (int b = 0; b < p.nbuf; ++b)
      for (uint32_t i = threadIdx.x * 16u; i < slack; i += kHaloWgradThreads * 16u)
        asm volatile("st.shared.v4.b32 [%0], {%1, %1, %1, %1};" ::"r"(smem_base + b * stage_bytes + halo_rows_bytes + i), "r"(0u)
                     : "memory");
    fence_proxy_async_smem();
  }
  __syncthreads();

  auto issue = [&](int strip, int b) {                     // (thread 0) halo tile + dY tile of `strip` into buffer b
    const int n = strip / p.strips_per_image, h0 = (strip % p.strips_per_image) * p.R;
    mbar_arrive_expect_tx(full_bar(b), p.a_tx_bytes + dy_bytes);
    const uint32_t x_dst = smem_base + b * stage_bytes;
    tma_load_4d(x_dst, &xmap, full_bar(b), 0, -1, h0 - 1, n);
    tma_load_4d(x_dst + p.a_buf_bytes, &dymap, full_bar(b), 0, 0, h0, n);
  };
  if (threadIdx.x == 0) {                                  // fill every buffer once
    int strip = blockIdx.x;
    for (int b = 0; b < p.nbuf && strip < p.total_strips; ++b, strip += gridDim.x) issue(strip, b);
  }
  {
    const int cw = warp;                                   // 0..11
    const int kh = cw >> 2, wq = cw & 3;                   // filter row; 16 input channels 16wq..16wq+15
    // ldmatrix.trans: lane supplies position (K) row 8 * (lane >> 4) + (lane & 7) of matrix lane / 8, whose 8
    // channels are chunk 2wq + ((lane >> 3) & 1) of the 128-byte row.
    const uint32_t lpos = (uint32_t)(8 * (lane >> 4) + (lane & 7));
    const uint32_t lchunk = (uint32_t)(2 * wq + ((lane >> 3) & 1)) * 16u;
    float acc[3][32];
#pragma unroll
    for (int kw = 0; kw < 3; ++kw) zero_acc(acc[kw]);
    uint32_t a[3][4];
    int buf = 0; uint32_t phase = 0;
    const int ksteps = p.R * p.Wp / 16;
    for (int strip = blockIdx.x; strip < p.total_strips; strip += gridDim.x) {
      mbar_wait(full_bar(buf), phase);
      const uint32_t x_src = smem_base + buf * stage_bytes;
      const uint64_t db0 = make_smem_desc(x_src + p.a_buf_bytes, 8192, 1024);
      const uint32_t a0 = x_src + (uint32_t)(kh * p.Wp + (int)lpos) * 128u + lchunk;   // row_off[3kh] = kh * Wp
#pragma unroll 2
      for (int k = 0; k < ksteps; ++k) {                   // 16 positions = +2048 B of x and of dY rows
        // the three taps of filter row kh as one wgmma group; its fragments are reloaded only after it retires
#pragma unroll
        for (int kw = 0; kw < 3; ++kw) ldmatrix_x4_trans(a[kw], swz128(a0 + (uint32_t)(16 * k + kw) * 128u));
        wgmma_fence();
#pragma unroll
        for (int kw = 0; kw < 3; ++kw) Wgmma<64>::rs<1>(acc[kw], a[kw], db0 + (uint64_t)(128 * k));
        wgmma_commit();
        wgmma_wait<0>();
#pragma unroll
        for (int kw = 0; kw < 3; ++kw) keep_frag(a[kw]);
      }
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) fence_regs(acc[kw]);
      __syncwarp();
      if (lane == 0) mbar_arrive(empty_bar(buf));
      if (threadIdx.x == 0) {                              // refill this buffer once all 12 warps have released it
        const int next = strip + p.nbuf * (int)gridDim.x;
        if (next < p.total_strips) {
          mbar_wait(empty_bar(buf), phase);
          issue(next, buf);
        }
      }
      __syncwarp();
      if (++buf == p.nbuf) { buf = 0; phase ^= 1u; }
    }
    float* part = p.wgrad_out + (size_t)blockIdx.x * 9 * p.ci * p.N;
#pragma unroll
    for (int kw = 0; kw < 3; ++kw) {
      const int tap = 3 * kh + kw;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int ci = 16 * wq + (lane >> 2) + 8 * h;
        if (ci >= p.ci) continue;
        float* dst_row = part + ((size_t)tap * p.ci + ci) * p.N;
#pragma unroll
        for (int jc = 0; jc < 8; ++jc) {
          const int co = 8 * jc + 2 * (lane & 3);                     // co is even and p.N % 8 == 0
          if (co < p.N) *reinterpret_cast<float2*>(dst_row + co) = make_float2(acc[kw][4 * jc + 2 * h], acc[kw][4 * jc + 2 * h + 1]);
        }
      }
    }
  }
}

// ----------------------------------------------------------------------------
// Host side
// ----------------------------------------------------------------------------

// Geometry the halo kernels cover; `kred` = reduction channels per tap (cin for fprop, cout for dgrad).
static bool halo_geom(const ConvGeom& g, int kred, HaloParams* p, size_t smem_fixed, int dy_tile) {
  if (!halo_enabled() || g.ksize != 3 || g.stride != 1 || g.pad != 1) return false;
  if (g.in_h != g.out_h || g.in_w != g.out_w || kred > 64 || kred % 8) return false;
  int wp = 8;
  while (wp < g.in_w + 2) wp *= 2;
  if (wp > 128 || g.in_w * 4 < wp * 3) return false;          // < 75 % useful positions: not worth it
  const int rt = 128 / wp;
  // Strip height R = rt*T and the number of halo tiles in flight.  One TMA box per strip means the
  // load pipeline is only as deep as the buffers: prefer >= 3 buffers (measured: the kernels are
  // load-latency bound with 2), then the tallest strip (smallest halo overhead (R+2)/R).
  int best_t = 0, best_nbuf = 0; long long best_cost = 0;
  for (int nbuf = 2; nbuf <= 4; ++nbuf)
    for (int t = 1; t <= 8; ++t) {
      const int r = rt * t;
      const size_t a_buf = ((size_t)((r + 2) * wp + 8) * 128 + 1023) / 1024 * 1024;
      const size_t need = smem_fixed + nbuf * (a_buf + (dy_tile ? (size_t)r * wp * 128 : 0)) + 2048;
      if (need > 227 * 1024) break;
      const long long strips = (g.in_h + r - 1) / r;
      // rows fetched + rows computed per image, scaled by a pipeline-depth penalty
      long long cost = (strips * (r + 2) + strips * r) * 16 + strips * 8;
      if (nbuf == 2) cost = cost * 3 / 2;
      if (best_t == 0 || cost < best_cost) { best_t = t; best_nbuf = nbuf; best_cost = cost; }
      if (r >= g.in_h) break;
    }
  if (best_t == 0) return false;
  p->W = g.in_w; p->H = g.in_h; p->NB = g.batch; p->Wp = wp;
  p->T = best_t; p->R = rt * best_t; p->nbuf = best_nbuf;
  p->strips_per_image = (g.in_h + p->R - 1) / p->R;
  p->total_strips = p->strips_per_image * g.batch;
  p->a_tx_bytes = (uint32_t)((p->R + 2) * wp) * 128u;
  p->a_buf_bytes = (uint32_t)(((size_t)((p->R + 2) * wp + 8) * 128 + 1023) / 1024 * 1024);
  return true;
}

static bool halo_fprop_ok(const ConvGeom& g, HaloParams* p) {
  return g.cout % 8 == 0 && g.x_pitch % 8 == 0 && halo_geom(g, g.cin, p, 9 * kHaloBTapBytes + 2 * kHaloSlabBytes, 0);
}
static bool halo_dgrad_ok(const ConvGeom& g, HaloParams* p) {
  return g.cin % 8 == 0 && g.x_pitch % 8 == 0 && halo_geom(g, g.cout, p, 9 * kHaloBTapBytes + 2 * kHaloSlabBytes, 0);
}
static bool halo_wgrad_ok(const ConvGeom& g, HaloParams* p) {
  return g.cout <= 64 && g.cout % 8 == 0 && g.x_pitch % 8 == 0 && halo_geom(g, g.cin, p, 0, 1);
}
static int halo_wgrad_grid(const HaloParams& p) {
  ensure_driver();
  const int sms = g_num_sms > 0 ? g_num_sms : kNumSmsHint;
  return p.total_strips < sms ? p.total_strips : sms;
}
static size_t halo_wgrad_ws_elems(const ConvGeom& g, const HaloParams& p) {
  return (size_t)halo_wgrad_grid(p) * 9 * g.cin * g.cout;
}

// in: activations [NB,H,W,kred] (pitch in_pitch); out: [NB,H,W,n_out] (pitch out_pitch);
// wts: packed [tap][n_out][kpad] K-major bf16; flip = dgrad (tap (kh,kw) reads the pixel at (1-kh, 1-kw));
// relu: k_halo3x3_kmajor_relu.
static int halo_launch_kmajor(HaloParams p, const void* in, int kred, int in_pitch, const void* wts, int kpad,
                              int n_out, void* out, int out_pitch, bool flip, cudaStream_t s, bool relu = false) {
  for (int kh = 0; kh < 3; ++kh)
    for (int kw = 0; kw < 3; ++kw) {
      const int t = kh * 3 + kw;
      const int dh = flip ? 1 - kh : kh - 1, dw = flip ? 1 - kw : kw - 1;
      p.row_off[t] = (dh + 1) * p.Wp + (dw + 1);
    }
  p.N = n_out;
  CUtensorMap amap, bmap, omap;
  const uint32_t abox[4] = {64, (uint32_t)p.Wp, (uint32_t)(p.R + 2), 1};
  int rc = make_act_map(&amap, in, p.NB, p.H, p.W, kred, in_pitch, 1, 0, 0, abox);
  if (rc != RIGL_OK) return rc;
  const uint64_t bdims[3] = {(uint64_t)kpad, (uint64_t)n_out, 9};
  const uint64_t bstr[2] = {(uint64_t)kpad * 2, (uint64_t)n_out * kpad * 2};
  const uint32_t bbox[3] = {64, 64, 1};
  rc = make_tmap(&bmap, wts, 3, bdims, bstr, bbox);
  if (rc != RIGL_OK) return rc;
  const uint32_t obox[4] = {64, (uint32_t)p.Wp, (uint32_t)(128 / p.Wp), 1};
  rc = make_act_map(&omap, out, p.NB, p.H, p.W, n_out, out_pitch, 1, 0, 0, obox);
  if (rc != RIGL_OK) return rc;
  const size_t smem = 9 * kHaloBTapBytes + p.nbuf * (size_t)p.a_buf_bytes + 2 * kHaloSlabBytes + 1024 + 256;
  RIGL_CUDA(relu ? smem_limit<k_halo3x3_kmajor_relu>(smem) : smem_limit<k_halo3x3_kmajor>(smem));
  auto kern = relu ? k_halo3x3_kmajor_relu : k_halo3x3_kmajor;
  const int n_tiles = (n_out + 63) / 64;
  const int sms = g_num_sms > 0 ? g_num_sms : kNumSmsHint;
  int gx = sms / n_tiles;
  if (gx < 1) gx = 1;
  if (gx > p.total_strips) gx = p.total_strips;
  kern<<<dim3((unsigned)gx, (unsigned)n_tiles), kThreads, smem, s>>>(amap, bmap, omap, p);
  RIGL_LAUNCH_CHECK(relu ? "k_halo3x3_kmajor_relu" : "k_halo3x3_kmajor");
  return RIGL_OK;
}

static int halo_launch_wgrad(HaloParams p, const ConvGeom& g, const void* x, const void* dy, float* partials,
                             cudaStream_t s) {
  for (int kh = 0; kh < 3; ++kh)
    for (int kw = 0; kw < 3; ++kw) {
      p.row_off[kh * 3 + kw] = kh * p.Wp + kw;
    }
  p.N = g.cout; p.ci = g.cin; p.wgrad_out = partials;
  CUtensorMap xmap, dymap;
  const uint32_t xbox[4] = {64, (uint32_t)p.Wp, (uint32_t)(p.R + 2), 1};
  int rc = make_act_map(&xmap, x, p.NB, p.H, p.W, g.cin, g.x_pitch, 1, 0, 0, xbox);
  if (rc != RIGL_OK) return rc;
  const uint32_t dbox[4] = {64, (uint32_t)p.Wp, (uint32_t)p.R, 1};
  rc = make_act_map(&dymap, dy, p.NB, p.H, p.W, g.cout, g.cout, 1, 0, 0, dbox);
  if (rc != RIGL_OK) return rc;
  const size_t smem = p.nbuf * ((size_t)p.a_buf_bytes + (size_t)p.R * p.Wp * 128) + 1024 + 256;
  RIGL_CUDA(smem_limit<k_halo3x3_wgrad>(smem));
  k_halo3x3_wgrad<<<(unsigned)halo_wgrad_grid(p), kHaloWgradThreads, smem, s>>>(xmap, dymap, p);
  RIGL_LAUNCH_CHECK("k_halo3x3_wgrad");
  return RIGL_OK;
}

