// Bitmap <-> float mask conversion, popcount, masked-gradient apply, and the
// library-wide error/launch bookkeeping.
#include <string.h>

#include "common.cuh"

namespace rigl {

std::atomic<uint64_t> g_launches{0};
static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

// One warp per 32-bit word: lane i owns element 32*word + i (coalesced).
__global__ void k_pack_f32(const float* __restrict__ src, int64_t n, uint32_t* __restrict__ bits,
                           int64_t words) {
  const int64_t word = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (word >= words) return;
  const int lane = threadIdx.x & 31;
  const int64_t e = word * 32 + lane;
  const bool on = e < n && src[e] != 0.0f;
  const uint32_t w = __ballot_sync(0xffffffffu, on);
  if (lane == 0) bits[word] = w;
}

__global__ void k_unpack_f32(const uint32_t* __restrict__ bits, int64_t n, float* __restrict__ dst) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < n) dst[e] = ((bits[e >> 5] >> (e & 31)) & 1u) ? 1.0f : 0.0f;
}

__global__ void k_popcount(const uint32_t* __restrict__ bits, int64_t words, int32_t* out) {
  uint32_t c = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < words;
       i += (int64_t)gridDim.x * blockDim.x)
    c += __popc(bits[i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, (int32_t)c);
}

// dst = bit ? src*scale : 0, float4 per thread (element e0 = 4*t).
__global__ void k_apply_mask_f32(const float* __restrict__ src, const uint32_t* __restrict__ bits,
                                 int64_t n, float* __restrict__ dst, float scale) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t e0 = t * 4;
  if (e0 >= n) return;
  const uint32_t nib = (bits[e0 >> 5] >> (e0 & 31)) & 0xFu;
  if (e0 + 3 < n) {
    float4 v = *reinterpret_cast<const float4*>(src + e0);
    v.x = (nib & 1u) ? v.x * scale : 0.f;
    v.y = (nib & 2u) ? v.y * scale : 0.f;
    v.z = (nib & 4u) ? v.z * scale : 0.f;
    v.w = (nib & 8u) ? v.w * scale : 0.f;
    *reinterpret_cast<float4*>(dst + e0) = v;
  } else {
    for (int c = 0; c < 4 && e0 + c < n; ++c) dst[e0 + c] = ((nib >> c) & 1u) ? src[e0 + c] * scale : 0.f;
  }
}

}  // namespace rigl

using namespace rigl;

extern "C" int rigl_version(void) { return 206; }
extern "C" const char* rigl_last_error(void) { return g_err; }
extern "C" uint64_t rigl_launch_count(void) { return g_launches.load(); }

extern "C" int rigl_mask_pack_f32(const float* src, int64_t n, uint32_t* bits, void* stream) {
  RIGL_REQUIRE(src && bits && n > 0, "rigl_mask_pack_f32: bad arguments");
  const int64_t words = rigl_mask_words(n);
  const int wpb = 8;
  k_pack_f32<<<(unsigned)((words + wpb - 1) / wpb), wpb * 32, 0, (cudaStream_t)stream>>>(src, n, bits, words);
  RIGL_LAUNCH_CHECK("k_pack_f32");
  return RIGL_OK;
}

extern "C" int rigl_mask_unpack_f32(const uint32_t* bits, int64_t n, float* dst, void* stream) {
  RIGL_REQUIRE(dst && bits && n > 0, "rigl_mask_unpack_f32: bad arguments");
  k_unpack_f32<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(bits, n, dst);
  RIGL_LAUNCH_CHECK("k_unpack_f32");
  return RIGL_OK;
}

extern "C" int rigl_mask_popcount(const uint32_t* bits, int64_t n, int32_t* out_count_dev, void* stream) {
  RIGL_REQUIRE(bits && out_count_dev && n > 0, "rigl_mask_popcount: bad arguments");
  const int64_t words = rigl_mask_words(n);
  RIGL_CUDA(cudaMemsetAsync(out_count_dev, 0, sizeof(int32_t), (cudaStream_t)stream));
  int blocks = (int)((words + 255) / 256);
  if (blocks > kNumSmsHint * 4) blocks = kNumSmsHint * 4;
  k_popcount<<<blocks, 256, 0, (cudaStream_t)stream>>>(bits, words, out_count_dev);
  RIGL_LAUNCH_CHECK("k_popcount");
  return RIGL_OK;
}

extern "C" int rigl_apply_mask_f32(const float* src, const uint32_t* bits, int64_t n, float* dst,
                                   float scale, void* stream) {
  RIGL_REQUIRE(src && bits && dst && n > 0, "rigl_apply_mask_f32: bad arguments");
  RIGL_REQUIRE(aligned16(src) && aligned16(dst), "rigl_apply_mask_f32: src/dst must be 16-byte aligned");
  const int64_t threads = (n + 3) / 4;
  k_apply_mask_f32<<<(unsigned)((threads + 255) / 256), 256, 0, (cudaStream_t)stream>>>(src, bits, n, dst, scale);
  RIGL_LAUNCH_CHECK("k_apply_mask_f32");
  return RIGL_OK;
}
