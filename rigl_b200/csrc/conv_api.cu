// C-ABI entry points of the masked conv / linear path: argument validation, then conv_route (igemm_tc.cu) picks
// the wgmma implicit-GEMM or halo kernels (igemm_tc.cu) or the CUDA-core kernels (conv_simt.cu).
#include <stdlib.h>

#include "common.cuh"
#include "conv_common.cuh"

namespace rigl {

static int g_force_simt = -1;

bool force_simt() {
  if (g_force_simt < 0) {
    const char* e = getenv("RIGL_FORCE_SIMT");
    g_force_simt = (e && e[0] == '1') ? 1 : 0;
  }
  return g_force_simt == 1;
}

int geom_from_desc(const rigl_conv_desc* d, ConvGeom* g) {
  RIGL_REQUIRE(d != nullptr, "null conv desc");
  RIGL_REQUIRE(d->batch > 0 && d->in_h > 0 && d->in_w > 0 && d->cin > 0 && d->cout > 0 && d->ksize > 0 &&
                   d->stride > 0 && d->pad >= 0,
               "conv desc: non-positive dimension");
  // `pad` is the padding BEFORE the image; windows may overrun the far edge (implicit zero
  // padding there), which covers TF 'SAME' (asymmetric for stride 2), explicit fixed padding
  // and 'VALID'.  Every window must start inside the padded image.
  RIGL_REQUIRE(d->pad < d->ksize && d->out_h > 0 && d->out_w > 0 &&
                   (d->out_h - 1) * d->stride - d->pad < d->in_h && (d->out_w - 1) * d->stride - d->pad < d->in_w,
               "conv desc: output %dx%d inconsistent with input %dx%d, k=%d, stride=%d, pad=%d", d->out_h,
               d->out_w, d->in_h, d->in_w, d->ksize, d->stride, d->pad);
  g->batch = d->batch; g->in_h = d->in_h; g->in_w = d->in_w; g->cin = d->cin;
  g->out_h = d->out_h; g->out_w = d->out_w; g->cout = d->cout;
  g->ksize = d->ksize; g->stride = d->stride; g->pad = d->pad;
  g->cin_pad = round_up8(d->cin); g->cout_pad = round_up8(d->cout);
  g->x_pitch = d->x_pitch > 0 ? d->x_pitch : d->cin;
  RIGL_REQUIRE(g->x_pitch >= d->cin, "conv desc: x_pitch %d < cin %d", g->x_pitch, d->cin);
  return RIGL_OK;
}

}  // namespace rigl

using namespace rigl;

extern "C" int rigl_im2col_nhwc(const rigl_conv_desc* d, const void* x, void* out, int64_t out_pitch,
                                void* stream) {
  ConvGeom g;
  int rc = geom_from_desc(d, &g);
  if (rc != RIGL_OK) return rc;
  RIGL_REQUIRE(x && out && out_pitch >= (int64_t)g.taps() * g.cin, "rigl_im2col_nhwc: bad arguments");
  return simt_im2col(g, x, out, out_pitch, (cudaStream_t)stream);
}

// ---- space-to-depth 7x7/2 stem (stem_s2d.cuh) ----
extern "C" int rigl_stem_s2d_supported(const rigl_conv_desc* d) {
  ConvGeom g;
  if (geom_from_desc(d, &g) != RIGL_OK) return 0;
  return s2d_supported(g) && !force_simt() ? 1 : 0;
}
extern "C" size_t rigl_stem_s2d_folded_bytes(const rigl_conv_desc* d) {
  ConvGeom g;
  return geom_from_desc(d, &g) == RIGL_OK ? s2d_folded_bytes(g) : 0;
}
extern "C" size_t rigl_stem_s2d_packed_bytes(const rigl_conv_desc* d) {
  ConvGeom g;
  return geom_from_desc(d, &g) == RIGL_OK ? s2d_packed_bytes(g) : 0;
}
extern "C" size_t rigl_stem_s2d_workspace_bytes(const rigl_conv_desc* d) {
  ConvGeom g;
  return geom_from_desc(d, &g) == RIGL_OK ? s2d_workspace_bytes(g) : 0;
}
extern "C" int rigl_stem_s2d_fold_input(const rigl_conv_desc* d, const void* x, void* xs, void* stream) {
  ConvGeom g;
  int rc = geom_from_desc(d, &g);
  if (rc != RIGL_OK) return rc;
  RIGL_REQUIRE(x && xs && s2d_supported(g) && aligned16(xs), "rigl_stem_s2d_fold_input: bad arguments");
  return s2d_fold(g, x, xs, (cudaStream_t)stream);
}
extern "C" int rigl_stem_s2d_pack_weights(const rigl_conv_desc* d, const float* w_hwio, const uint32_t* mask_bits,
                                          void* packed, void* stream) {
  ConvGeom g;
  int rc = geom_from_desc(d, &g);
  if (rc != RIGL_OK) return rc;
  RIGL_REQUIRE(w_hwio && mask_bits && packed && s2d_supported(g), "rigl_stem_s2d_pack_weights: bad arguments");
  return s2d_pack(g, w_hwio, mask_bits, packed, (cudaStream_t)stream);
}
extern "C" int rigl_stem_s2d_fprop(const rigl_conv_desc* d, const void* xs, const void* packed, void* y,
                                   void* stream) {
  ConvGeom g;
  int rc = geom_from_desc(d, &g);
  if (rc != RIGL_OK) return rc;
  RIGL_REQUIRE(xs && packed && y && s2d_supported(g), "rigl_stem_s2d_fprop: bad arguments");
  return s2d_fprop(g, xs, packed, y, (cudaStream_t)stream);
}
extern "C" int rigl_stem_s2d_wgrad(const rigl_conv_desc* d, const void* xs, const void* dy, float* dw, float beta,
                                   void* ws, size_t ws_bytes, void* stream) {
  ConvGeom g;
  int rc = geom_from_desc(d, &g);
  if (rc != RIGL_OK) return rc;
  RIGL_REQUIRE(xs && dy && dw && s2d_supported(g), "rigl_stem_s2d_wgrad: bad arguments");
  return s2d_wgrad(g, xs, dy, dw, beta, ws, ws_bytes, (cudaStream_t)stream);
}

extern "C" int rigl_set_force_simt(int on) {
  g_force_simt = on ? 1 : 0;
  return RIGL_OK;
}

extern "C" size_t rigl_conv_workspace_bytes(const rigl_conv_desc* d) {
  ConvGeom g;
  if (geom_from_desc(d, &g) != RIGL_OK) return 0;
  return tc_workspace_bytes(g);
}

// Routes one fprop / dgrad and runs it.  The CUDA-core fprop reads the dgrad-layout weights of the packed blob, the
// CUDA-core dgrad the fprop-layout ones.
static int run_fprop(const ConvGeom& g, const void* x, const void* packed, void* y, const ConvEpilogue& epi,
                     void* stream) {
  const int path = conv_route(g, 0, epi);
  if (path < 0) return path;
  if (path == kPathSimt)
    return simt_fprop(g, x, static_cast<const uint8_t*>(packed) + packed_layout(g.taps(), g.cin, g.cout).off_dgrad, y,
                      epi.out_f32, epi.bias, (cudaStream_t)stream);
  return tc_fprop(g, path, x, packed, y, epi, (cudaStream_t)stream);
}

static int run_dgrad(const ConvGeom& g, const void* dy, const void* packed, void* dx, const ConvEpilogue& epi,
                     void* stream) {
  const int path = conv_route(g, 1, epi);
  if (path < 0) return path;
  if (path == kPathSimt)
    return simt_dgrad(g, dy, static_cast<const uint8_t*>(packed) + packed_layout(g.taps(), g.cin, g.cout).off_fprop,
                      dx, (cudaStream_t)stream);
  return tc_dgrad(g, path, dy, packed, dx, epi, (cudaStream_t)stream);
}

extern "C" int rigl_masked_conv2d_fprop(const rigl_conv_desc* d, const void* x, const void* packed,
                                        void* y_bf16, float* y_f32, const float* bias, void* ws,
                                        size_t ws_bytes, void* stream) {
  ConvGeom g;
  int rc = geom_from_desc(d, &g);
  if (rc != RIGL_OK) return rc;
  RIGL_REQUIRE(x && packed && (y_bf16 || y_f32), "rigl_masked_conv2d_fprop: null tensor");
  ConvEpilogue epi;
  epi.out_f32 = y_f32; epi.bias = bias;
  return run_fprop(g, x, packed, y_bf16, epi, stream);
}

extern "C" int rigl_bn_partial_rows(void) { return tc_max_ctas(); }

extern "C" int rigl_set_bn_stats_always(int on) {
  tc_set_bn_stats_always(on != 0);
  return RIGL_OK;
}

extern "C" int rigl_masked_conv2d_fprop_bnstats(const rigl_conv_desc* d, const void* x, const void* packed,
                                                void* y_bf16, float* bn_partial, int* bn_rows_out, void* ws,
                                                size_t ws_bytes, void* stream) {
  ConvGeom g;
  int rc = geom_from_desc(d, &g);
  if (rc != RIGL_OK) return rc;
  RIGL_REQUIRE(x && packed && y_bf16 && bn_partial && bn_rows_out, "rigl_masked_conv2d_fprop_bnstats: null argument");
  ConvEpilogue epi;
  epi.kind = ConvEpilogue::kBnStats;
  epi.bn_partial = bn_partial; epi.bn_rows = bn_rows_out;
  return run_fprop(g, x, packed, y_bf16, epi, stream);
}

extern "C" int rigl_masked_conv2d_fprop_bnapply(const rigl_conv_desc* d, const void* x, const void* packed,
                                                const void* residual, const float* scale, const float* shift, int relu,
                                                void* y_bf16, void* ws, size_t ws_bytes, void* stream) {
  ConvGeom g;
  int rc = geom_from_desc(d, &g);
  if (rc != RIGL_OK) return rc;
  RIGL_REQUIRE(x && packed && scale && shift && y_bf16, "rigl_masked_conv2d_fprop_bnapply: null argument");
  RIGL_REQUIRE(g.cout % 8 == 0, "rigl_masked_conv2d_fprop_bnapply: cout %d is not a multiple of 8", g.cout);
  RIGL_REQUIRE(aligned16(x) && aligned16(y_bf16) && aligned16(residual),
               "rigl_masked_conv2d_fprop_bnapply: tensors must be 16-byte aligned");
  ConvEpilogue epi;
  epi.kind = ConvEpilogue::kBnApply;
  epi.residual = residual; epi.scale = scale; epi.shift = shift; epi.relu = relu;
  return run_fprop(g, x, packed, y_bf16, epi, stream);
}

extern "C" int rigl_masked_conv2d_fprop_relu(const rigl_conv_desc* d, const void* x, const void* packed, void* y_bf16,
                                             void* ws, size_t ws_bytes, void* stream) {
  ConvGeom g;
  int rc = geom_from_desc(d, &g);
  if (rc != RIGL_OK) return rc;
  RIGL_REQUIRE(x && packed && y_bf16, "rigl_masked_conv2d_fprop_relu: null argument");
  RIGL_REQUIRE(g.cout % 8 == 0, "rigl_masked_conv2d_fprop_relu: cout %d is not a multiple of 8", g.cout);
  RIGL_REQUIRE(aligned16(x) && aligned16(y_bf16), "rigl_masked_conv2d_fprop_relu: tensors must be 16-byte aligned");
  ConvEpilogue epi;
  epi.kind = ConvEpilogue::kRelu;
  return run_fprop(g, x, packed, y_bf16, epi, stream);
}

extern "C" int rigl_masked_conv2d_dgrad_relu(const rigl_conv_desc* d, const void* dy, const void* packed,
                                             const void* x, void* dx, void* ws, size_t ws_bytes, void* stream) {
  ConvGeom g;
  int rc = geom_from_desc(d, &g);
  if (rc != RIGL_OK) return rc;
  RIGL_REQUIRE(dy && packed && x && dx, "rigl_masked_conv2d_dgrad_relu: null argument");
  RIGL_REQUIRE(g.cin % 8 == 0 && g.cout % 8 == 0 && g.x_pitch % 8 == 0,
               "rigl_masked_conv2d_dgrad_relu: cin %d, cout %d and x_pitch %d must be multiples of 8", g.cin, g.cout,
               g.x_pitch);
  RIGL_REQUIRE(aligned16(dy) && aligned16(x) && aligned16(dx),
               "rigl_masked_conv2d_dgrad_relu: tensors must be 16-byte aligned");
  ConvEpilogue epi;
  epi.kind = ConvEpilogue::kReluGate;
  epi.gate = x;
  return run_dgrad(g, dy, packed, dx, epi, stream);
}

extern "C" int rigl_masked_conv2d_dgrad(const rigl_conv_desc* d, const void* dy, const void* packed,
                                        void* dx, void* ws, size_t ws_bytes, void* stream) {
  ConvGeom g;
  int rc = geom_from_desc(d, &g);
  if (rc != RIGL_OK) return rc;
  RIGL_REQUIRE(dy && packed && dx, "rigl_masked_conv2d_dgrad: null tensor");
  return run_dgrad(g, dy, packed, dx, ConvEpilogue(), stream);
}

extern "C" int rigl_conv2d_wgrad_dense(const rigl_conv_desc* d, const void* x, const void* dy, float* dw,
                                       float beta, void* ws, size_t ws_bytes, void* stream) {
  ConvGeom g;
  int rc = geom_from_desc(d, &g);
  if (rc != RIGL_OK) return rc;
  RIGL_REQUIRE(x && dy && dw, "rigl_conv2d_wgrad_dense: null tensor");
  RIGL_REQUIRE(beta == 0.f || beta == 1.f, "rigl_conv2d_wgrad_dense: beta must be 0 or 1");
  const int path = conv_route(g, 2, ConvEpilogue());
  if (path == kPathSimt) return simt_wgrad(g, x, dy, dw, beta, (cudaStream_t)stream);
  return tc_wgrad(g, path, x, dy, dw, beta, ws, ws_bytes, (cudaStream_t)stream);
}
