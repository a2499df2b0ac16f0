// Batched optimizer steps for ALL parameters of a model in one launch, with `mask * dense_grad` fused into the
// gradient load of the masked layers.  Two inner optimizers of the reference's training drivers share the task
// table, the descriptor upload and the alignment test below.
//
// Nesterov momentum.  Reference call site: imagenet_train_eval.py:355-365 -- tf.train.MomentumOptimizer(lr,
// momentum, use_nesterov=True) under the sparse wrapper, l2 regularisation on the raw weights;
// sparse_optimizers_base.py:478-485 hands it dL/dweights = mask * dL/d(mask*weights).  Per element
//   g     = (bit ? dense_grad * grad_scale : 0) + weight_decay * w          (grad_scale = 1/world under DP)
//   accum = momentum * accum + g
//   w    -= lr * (nesterov ? g + momentum * accum : accum)
// The learning rate is read from DEVICE memory, so a captured CUDA graph follows a schedule without re-capture.
// Before: one mask*grad kernel per layer (54) + five multi-tensor kernels over every parameter; now one pass that
// reads w, accum, grad (+ 1 bit) and writes w, accum: 20.125 bytes per masked weight.
//
// Adam.  Reference call sites: imagenet_train_eval.py:355-358 (--use_adam), mnist_train_eval.py:247-261,
// rigl_tf2/utils.py:get_optimizer -- tf.train.AdamOptimizer, i.e. TF 1.x ApplyAdam (use_nesterov=false) with the
// epsilon added to sqrt(v) BEFORE the bias correction (Kingma & Ba's eps-hat; torch.optim.Adam adds it after).
// Per element, every operation rounded once (no FMA contraction) so a numpy restatement matches bit for bit:
//   g     = (bit ? dense_grad * grad_scale : 0) + weight_decay * w
//   alpha = lr * sqrt(1 - beta2_power) / (1 - beta1_power)                 (once per block, device scalars)
//   m     = m + (g - m) * (1 - beta1)
//   v     = v + (g * g - v) * (1 - beta2)
//   w     = w - (m * alpha) / (sqrt(v) + epsilon)
// then, in a one-thread launch on the same stream, beta1_power *= beta1 and beta2_power *= beta2 (TF's _finish),
// so a captured step replays with no host work.  Reads w, m, v, grad (+ 1 bit), writes w, m, v: 28.125 bytes per
// masked weight.
//
// Training summaries.  Reference: train_function's scalars (imagenet_train_eval.py:431-470): grad_norm, var_norm,
// fw_nz_* and the mask sparsities.  On the same task table, per element
//   g = (bit ? dense_grad * grad_scale : 0) + reg_decay * w          (the optimizers' g, float32)
// and per task, in float64 from the element on: sum w^2, sum g^2, sum |w|, nnz(w) (NaN counts, +-0 does not) and
// the number of set bits of its elements.  A second launch adds each parameter's task rows in task order, so the
// result is bit-identical run to run.  Reads w, grad (+ 1 bit): 8.125 bytes per masked weight.
#include <initializer_list>
#include <vector>

#include "common.cuh"

namespace rigl {

constexpr int kSgdThreads = 256;
constexpr int kSgdChunk = 8192;          // elements per block

struct SgdLayerDev {
  float* p;
  float* m;
  const float* g;
  const uint32_t* bits;
  uint32_t n;
  float wd, gscale;
  uint32_t vec_ok;       // every pointer 16-byte aligned
};

// One block per kSgdChunk elements of one parameter (every batched optimizer kernel).
struct SgdTask { uint32_t layer, start; };

inline void append_tasks(std::vector<SgdTask>& tasks, int layer, int64_t n) {
  for (int64_t s = 0; s < n; s += kSgdChunk) tasks.push_back({(uint32_t)layer, (uint32_t)s});
}

// The float4 path is taken only when every pointer of a parameter is 16-byte aligned.
inline uint32_t vec_ok(std::initializer_list<const void*> ptrs) {
  for (const void* p : ptrs)
    if (!aligned16(p)) return 0u;
  return 1u;
}

// Device copies of a batched optimizer's layer table and task table.
template <class LayerDev>
struct BatchedPlan {
  int n_tasks = 0;
  LayerDev* d_layers = nullptr;
  SgdTask* d_tasks = nullptr;
};

template <class Plan, class LayerDev>
int upload_plan(const std::vector<LayerDev>& host, const std::vector<SgdTask>& tasks, Plan** out, const char* what) {
  Plan* p = new Plan();
  p->n_tasks = (int)tasks.size();
  cudaError_t e = cudaMalloc(&p->d_layers, sizeof(LayerDev) * host.size());
  if (e == cudaSuccess) e = cudaMalloc(&p->d_tasks, sizeof(SgdTask) * tasks.size());
  if (e == cudaSuccess) e = cudaMemcpy(p->d_layers, host.data(), sizeof(LayerDev) * host.size(), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(p->d_tasks, tasks.data(), sizeof(SgdTask) * tasks.size(), cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    cudaFree(p->d_layers); cudaFree(p->d_tasks); delete p;
    return cuda_fail(e, what);
  }
  *out = p;
  return RIGL_OK;
}

template <class Plan>
int destroy_plan(Plan* plan) {
  if (!plan) return RIGL_OK;
  cudaFree(plan->d_layers);
  cudaFree(plan->d_tasks);
  delete plan;
  return RIGL_OK;
}

__device__ __forceinline__ void sgd_one(float& p, float& m, float g, bool on, float wd, float gscale, float lr,
                                        float mom, int nesterov) {
  const float ge = fmaf(wd, p, on ? g * gscale : 0.f);
  m = fmaf(mom, m, ge);
  p = fmaf(-lr, nesterov ? fmaf(mom, m, ge) : m, p);
}

__global__ void __launch_bounds__(kSgdThreads)
k_sgd_nesterov_batched(const SgdLayerDev* __restrict__ layers, const SgdTask* __restrict__ tasks,
                       const float* __restrict__ lr_dev, float mom, int nesterov) {
  const SgdTask t = tasks[blockIdx.x];
  const SgdLayerDev L = layers[t.layer];
  const float lr = __ldg(lr_dev);
  const uint32_t end = min(L.n, t.start + (uint32_t)kSgdChunk);
  if (L.vec_ok) {
#pragma unroll 2
    for (uint32_t e = t.start + 4 * threadIdx.x; e < end; e += 4 * kSgdThreads) {
      if (e + 3 < L.n) {
        float4 p = *reinterpret_cast<const float4*>(L.p + e);
        float4 m = *reinterpret_cast<const float4*>(L.m + e);
        const float4 g = __ldg(reinterpret_cast<const float4*>(L.g + e));
        const uint32_t nib = L.bits ? (__ldg(L.bits + (e >> 5)) >> (e & 31)) & 0xFu : 0xFu;
        sgd_one(p.x, m.x, g.x, nib & 1u, L.wd, L.gscale, lr, mom, nesterov);
        sgd_one(p.y, m.y, g.y, nib & 2u, L.wd, L.gscale, lr, mom, nesterov);
        sgd_one(p.z, m.z, g.z, nib & 4u, L.wd, L.gscale, lr, mom, nesterov);
        sgd_one(p.w, m.w, g.w, nib & 8u, L.wd, L.gscale, lr, mom, nesterov);
        *reinterpret_cast<float4*>(L.p + e) = p;
        *reinterpret_cast<float4*>(L.m + e) = m;
      } else {
        for (uint32_t j = e; j < L.n; ++j) {
          const bool on = L.bits ? (__ldg(L.bits + (j >> 5)) >> (j & 31)) & 1u : true;
          sgd_one(L.p[j], L.m[j], __ldg(L.g + j), on, L.wd, L.gscale, lr, mom, nesterov);
        }
      }
    }
  } else {
    for (uint32_t j = t.start + threadIdx.x; j < end; j += kSgdThreads) {
      const bool on = L.bits ? (__ldg(L.bits + (j >> 5)) >> (j & 31)) & 1u : true;
      sgd_one(L.p[j], L.m[j], __ldg(L.g + j), on, L.wd, L.gscale, lr, mom, nesterov);
    }
  }
}

struct AdamLayerDev {
  float* p;
  float* m;
  float* v;
  const float* g;
  const uint32_t* bits;
  uint32_t n;
  float wd, gscale;
  uint32_t vec_ok;       // every pointer 16-byte aligned
};

struct AdamCoef { float alpha, omb1, omb2, eps; };

__device__ __forceinline__ void adam_one(float& p, float& m, float& v, float g, bool on, float wd, float gscale,
                                         const AdamCoef& c) {
  const float ge = __fadd_rn(on ? __fmul_rn(g, gscale) : 0.f, __fmul_rn(wd, p));
  m = __fadd_rn(m, __fmul_rn(__fsub_rn(ge, m), c.omb1));
  v = __fadd_rn(v, __fmul_rn(__fsub_rn(__fmul_rn(ge, ge), v), c.omb2));
  p = __fsub_rn(p, __fdiv_rn(__fmul_rn(m, c.alpha), __fadd_rn(__fsqrt_rn(v), c.eps)));
}

__global__ void __launch_bounds__(kSgdThreads)
k_adam_batched(const AdamLayerDev* __restrict__ layers, const SgdTask* __restrict__ tasks,
               const float* __restrict__ lr_dev, const float* __restrict__ powers, float beta1, float beta2,
               float eps) {
  const SgdTask t = tasks[blockIdx.x];
  const AdamLayerDev L = layers[t.layer];
  AdamCoef c;
  c.alpha = __fdiv_rn(__fmul_rn(__ldg(lr_dev), __fsqrt_rn(__fsub_rn(1.f, powers[1]))), __fsub_rn(1.f, powers[0]));
  c.omb1 = __fsub_rn(1.f, beta1);
  c.omb2 = __fsub_rn(1.f, beta2);
  c.eps = eps;
  const uint32_t end = min(L.n, t.start + (uint32_t)kSgdChunk);
  if (L.vec_ok) {
#pragma unroll 2
    for (uint32_t e = t.start + 4 * threadIdx.x; e < end; e += 4 * kSgdThreads) {
      if (e + 3 < L.n) {
        float4 p = *reinterpret_cast<const float4*>(L.p + e);
        float4 m = *reinterpret_cast<const float4*>(L.m + e);
        float4 v = *reinterpret_cast<const float4*>(L.v + e);
        const float4 g = __ldg(reinterpret_cast<const float4*>(L.g + e));
        const uint32_t nib = L.bits ? (__ldg(L.bits + (e >> 5)) >> (e & 31)) & 0xFu : 0xFu;
        adam_one(p.x, m.x, v.x, g.x, nib & 1u, L.wd, L.gscale, c);
        adam_one(p.y, m.y, v.y, g.y, nib & 2u, L.wd, L.gscale, c);
        adam_one(p.z, m.z, v.z, g.z, nib & 4u, L.wd, L.gscale, c);
        adam_one(p.w, m.w, v.w, g.w, nib & 8u, L.wd, L.gscale, c);
        *reinterpret_cast<float4*>(L.p + e) = p;
        *reinterpret_cast<float4*>(L.m + e) = m;
        *reinterpret_cast<float4*>(L.v + e) = v;
      } else {
        for (uint32_t j = e; j < L.n; ++j) {
          const bool on = L.bits ? (__ldg(L.bits + (j >> 5)) >> (j & 31)) & 1u : true;
          adam_one(L.p[j], L.m[j], L.v[j], __ldg(L.g + j), on, L.wd, L.gscale, c);
        }
      }
    }
  } else {
    for (uint32_t j = t.start + threadIdx.x; j < end; j += kSgdThreads) {
      const bool on = L.bits ? (__ldg(L.bits + (j >> 5)) >> (j & 31)) & 1u : true;
      adam_one(L.p[j], L.m[j], L.v[j], __ldg(L.g + j), on, L.wd, L.gscale, c);
    }
  }
}

// After every block of k_adam_batched has read the powers (stream order): TF's _finish.
__global__ void k_adam_advance_powers(float* powers, float beta1, float beta2) {
  powers[0] = __fmul_rn(powers[0], beta1);
  powers[1] = __fmul_rn(powers[1], beta2);
}

struct SummaryLayerDev {
  const float* p;
  const float* g;
  const uint32_t* bits;
  uint32_t n;
  float reg_decay, gscale;
  uint32_t vec_ok;       // both pointers 16-byte aligned
  uint32_t task0;        // index of the parameter's first task
};

// Columns of a partial row and of a result row.
constexpr int kSumW2 = 0, kSumG2 = 1, kSumAbsW = 2, kNnzW = 3, kOnes = 4, kSummaryCols = 5;

struct SummaryAcc {
  double w2 = 0.0, g2 = 0.0, l1 = 0.0;
  uint32_t nnz = 0, ones = 0;
};

__device__ __forceinline__ void summary_one(SummaryAcc& a, float w, float g, bool on, float rd, float gscale) {
  const float ge = fmaf(rd, w, on ? g * gscale : 0.f);     // sgd_one's g, reg_decay in place of weight_decay
  const double wd = w, gd = ge;
  a.w2 = fma(wd, wd, a.w2);
  a.g2 = fma(gd, gd, a.g2);
  a.l1 += fabs(wd);
  a.nnz += w != 0.f;
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// One block per task: one partial row [kSummaryCols] per task.  The reduction tree is fixed (butterfly within a
// warp, then warps in order), so a row is the same on every run.
__global__ void __launch_bounds__(kSgdThreads)
k_train_summary(const SummaryLayerDev* __restrict__ layers, const SgdTask* __restrict__ tasks,
                double* __restrict__ partials) {
  const SgdTask t = tasks[blockIdx.x];
  const SummaryLayerDev L = layers[t.layer];
  const uint32_t end = min(L.n, t.start + (uint32_t)kSgdChunk);
  SummaryAcc a;
  if (L.vec_ok) {
#pragma unroll 2
    for (uint32_t e = t.start + 4 * threadIdx.x; e < end; e += 4 * kSgdThreads) {
      if (e + 3 < L.n) {
        const float4 p = __ldg(reinterpret_cast<const float4*>(L.p + e));
        const float4 g = __ldg(reinterpret_cast<const float4*>(L.g + e));
        const uint32_t nib = L.bits ? (__ldg(L.bits + (e >> 5)) >> (e & 31)) & 0xFu : 0xFu;
        summary_one(a, p.x, g.x, nib & 1u, L.reg_decay, L.gscale);
        summary_one(a, p.y, g.y, nib & 2u, L.reg_decay, L.gscale);
        summary_one(a, p.z, g.z, nib & 4u, L.reg_decay, L.gscale);
        summary_one(a, p.w, g.w, nib & 8u, L.reg_decay, L.gscale);
        if (L.bits) a.ones += __popc(nib);
      } else {
        for (uint32_t j = e; j < L.n; ++j) {
          const bool on = L.bits ? (__ldg(L.bits + (j >> 5)) >> (j & 31)) & 1u : true;
          summary_one(a, __ldg(L.p + j), __ldg(L.g + j), on, L.reg_decay, L.gscale);
          if (L.bits) a.ones += on;
        }
      }
    }
  } else {
    for (uint32_t j = t.start + threadIdx.x; j < end; j += kSgdThreads) {
      const bool on = L.bits ? (__ldg(L.bits + (j >> 5)) >> (j & 31)) & 1u : true;
      summary_one(a, __ldg(L.p + j), __ldg(L.g + j), on, L.reg_decay, L.gscale);
      if (L.bits) a.ones += on;
    }
  }
  // counts are at most kSgdChunk: exact in a double
  double v[kSummaryCols] = {a.w2, a.g2, a.l1, (double)a.nnz, (double)a.ones};
  __shared__ double s[kSgdThreads / 32][kSummaryCols];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int c = 0; c < kSummaryCols; ++c) {
    v[c] = warp_sum(v[c]);
    if (lane == 0) s[warp][c] = v[c];
  }
  __syncthreads();
  if (threadIdx.x < kSummaryCols) {
    double r = 0.0;
#pragma unroll
    for (int w = 0; w < kSgdThreads / 32; ++w) r += s[w][threadIdx.x];
    partials[(size_t)blockIdx.x * kSummaryCols + threadIdx.x] = r;
  }
}

// One block per parameter: its task rows, staged through shared memory, added in task order per column.
__global__ void __launch_bounds__(kSgdThreads)
k_train_summary_finalize(const SummaryLayerDev* __restrict__ layers, const double* __restrict__ partials,
                         double* __restrict__ out) {
  const SummaryLayerDev L = layers[blockIdx.x];
  const uint32_t n_tasks = (L.n + kSgdChunk - 1) / kSgdChunk;
  __shared__ double rows[kSgdThreads * kSummaryCols];
  double r = 0.0;
  for (uint32_t base = 0; base < n_tasks; base += kSgdThreads) {
    const uint32_t cnt = min(n_tasks - base, (uint32_t)kSgdThreads);
    const double* src = partials + (size_t)(L.task0 + base) * kSummaryCols;
    for (uint32_t i = threadIdx.x; i < cnt * kSummaryCols; i += kSgdThreads) rows[i] = src[i];
    __syncthreads();
    if (threadIdx.x < kSummaryCols)
      for (uint32_t k = 0; k < cnt; ++k) r += rows[k * kSummaryCols + threadIdx.x];
    __syncthreads();
  }
  if (threadIdx.x < kSummaryCols) out[(size_t)blockIdx.x * kSummaryCols + threadIdx.x] = r;
}

}  // namespace rigl

struct rigl_sgd_plan : rigl::BatchedPlan<rigl::SgdLayerDev> {};
struct rigl_adam_plan : rigl::BatchedPlan<rigl::AdamLayerDev> {};
struct rigl_summary_plan : rigl::BatchedPlan<rigl::SummaryLayerDev> {
  int n_params = 0;
  double* d_partials = nullptr;    // [n_tasks][kSummaryCols]
};

using namespace rigl;

extern "C" int rigl_sgd_plan_create(const rigl_sgd_desc* params, int n_params, rigl_sgd_plan** out) {
  RIGL_REQUIRE(params && out && n_params > 0, "rigl_sgd_plan_create: bad arguments");
  std::vector<SgdLayerDev> host(n_params);
  std::vector<SgdTask> tasks;
  for (int i = 0; i < n_params; ++i) {
    const rigl_sgd_desc& d = params[i];
    RIGL_REQUIRE(d.param && d.momentum && d.grad && d.n >= 1 && d.n < (1ll << 31),
                 "rigl_sgd_plan_create: parameter %d: null tensor or bad size", i);
    RIGL_REQUIRE((reinterpret_cast<uintptr_t>(d.param) & 3) == 0 && (reinterpret_cast<uintptr_t>(d.momentum) & 3) == 0 &&
                     (reinterpret_cast<uintptr_t>(d.grad) & 3) == 0, "parameter %d: tensors must be float-aligned", i);
    SgdLayerDev& L = host[i];
    L.p = d.param; L.m = d.momentum; L.g = d.grad; L.bits = d.mask_bits; L.n = (uint32_t)d.n;
    L.wd = d.weight_decay; L.gscale = d.grad_scale;
    L.vec_ok = vec_ok({d.param, d.momentum, d.grad});
    append_tasks(tasks, i, d.n);
  }
  return upload_plan(host, tasks, out, "rigl_sgd_plan_create");
}

extern "C" int rigl_sgd_plan_destroy(rigl_sgd_plan* plan) { return destroy_plan(plan); }

extern "C" int rigl_sgd_plan_run(rigl_sgd_plan* plan, const float* lr_dev, float momentum, int nesterov,
                                 void* stream_) {
  RIGL_REQUIRE(plan && lr_dev, "rigl_sgd_plan_run: null argument");
  k_sgd_nesterov_batched<<<plan->n_tasks, kSgdThreads, 0, (cudaStream_t)stream_>>>(plan->d_layers, plan->d_tasks, lr_dev,
                                                                                 momentum, nesterov ? 1 : 0);
  RIGL_LAUNCH_CHECK("k_sgd_nesterov_batched");
  return RIGL_OK;
}

extern "C" int rigl_adam_plan_create(const rigl_adam_desc* params, int n_params, rigl_adam_plan** out) {
  RIGL_REQUIRE(params && out && n_params > 0, "rigl_adam_plan_create: bad arguments");
  std::vector<AdamLayerDev> host(n_params);
  std::vector<SgdTask> tasks;
  for (int i = 0; i < n_params; ++i) {
    const rigl_adam_desc& d = params[i];
    RIGL_REQUIRE(d.param && d.m && d.v && d.grad && d.n >= 1 && d.n < (1ll << 31),
                 "rigl_adam_plan_create: parameter %d: null tensor or bad size", i);
    RIGL_REQUIRE(((reinterpret_cast<uintptr_t>(d.param) | reinterpret_cast<uintptr_t>(d.m) |
                   reinterpret_cast<uintptr_t>(d.v) | reinterpret_cast<uintptr_t>(d.grad)) & 3) == 0,
                 "rigl_adam_plan_create: parameter %d: tensors must be float-aligned", i);
    AdamLayerDev& L = host[i];
    L.p = d.param; L.m = d.m; L.v = d.v; L.g = d.grad; L.bits = d.mask_bits; L.n = (uint32_t)d.n;
    L.wd = d.weight_decay; L.gscale = d.grad_scale;
    L.vec_ok = vec_ok({d.param, d.m, d.v, d.grad});
    append_tasks(tasks, i, d.n);
  }
  return upload_plan(host, tasks, out, "rigl_adam_plan_create");
}

extern "C" int rigl_adam_plan_destroy(rigl_adam_plan* plan) { return destroy_plan(plan); }

extern "C" int rigl_adam_plan_run(rigl_adam_plan* plan, const float* lr_dev, float* powers_dev, float beta1,
                                  float beta2, float epsilon, void* stream_) {
  RIGL_REQUIRE(plan && lr_dev && powers_dev, "rigl_adam_plan_run: null argument");
  RIGL_REQUIRE(beta1 >= 0.f && beta1 < 1.f && beta2 >= 0.f && beta2 < 1.f && epsilon >= 0.f,
               "rigl_adam_plan_run: need 0 <= beta1, beta2 < 1 and epsilon >= 0");
  const cudaStream_t stream = (cudaStream_t)stream_;
  k_adam_batched<<<plan->n_tasks, kSgdThreads, 0, stream>>>(plan->d_layers, plan->d_tasks, lr_dev, powers_dev, beta1,
                                                             beta2, epsilon);
  RIGL_LAUNCH_CHECK("k_adam_batched");
  k_adam_advance_powers<<<1, 1, 0, stream>>>(powers_dev, beta1, beta2);
  RIGL_LAUNCH_CHECK("k_adam_advance_powers");
  return RIGL_OK;
}

extern "C" int rigl_summary_plan_create(const rigl_summary_desc* params, int n_params, rigl_summary_plan** out) {
  RIGL_REQUIRE(params && out && n_params > 0, "rigl_summary_plan_create: bad arguments");
  std::vector<SummaryLayerDev> host(n_params);
  std::vector<SgdTask> tasks;
  for (int i = 0; i < n_params; ++i) {
    const rigl_summary_desc& d = params[i];
    RIGL_REQUIRE(d.param && d.grad && d.n >= 1 && d.n < (1ll << 31),
                 "rigl_summary_plan_create: parameter %d: null tensor or bad size", i);
    RIGL_REQUIRE(((reinterpret_cast<uintptr_t>(d.param) | reinterpret_cast<uintptr_t>(d.grad)) & 3) == 0,
                 "rigl_summary_plan_create: parameter %d: tensors must be float-aligned", i);
    SummaryLayerDev& L = host[i];
    L.p = d.param; L.g = d.grad; L.bits = d.mask_bits; L.n = (uint32_t)d.n;
    L.reg_decay = d.reg_decay; L.gscale = d.grad_scale;
    L.vec_ok = vec_ok({d.param, d.grad});
    L.task0 = (uint32_t)tasks.size();
    append_tasks(tasks, i, d.n);
  }
  rigl_summary_plan* plan = nullptr;
  const int rc = upload_plan(host, tasks, &plan, "rigl_summary_plan_create");
  if (rc != RIGL_OK) return rc;
  plan->n_params = n_params;
  const cudaError_t e = cudaMalloc(&plan->d_partials, sizeof(double) * kSummaryCols * tasks.size());
  if (e != cudaSuccess) {
    destroy_plan(plan);
    return cuda_fail(e, "rigl_summary_plan_create");
  }
  *out = plan;
  return RIGL_OK;
}

extern "C" int rigl_summary_plan_destroy(rigl_summary_plan* plan) {
  if (plan) cudaFree(plan->d_partials);
  return destroy_plan(plan);
}

extern "C" int rigl_summary_plan_run(rigl_summary_plan* plan, double* out_dev, void* stream_) {
  RIGL_REQUIRE(plan && out_dev, "rigl_summary_plan_run: null argument");
  const cudaStream_t stream = (cudaStream_t)stream_;
  k_train_summary<<<plan->n_tasks, kSgdThreads, 0, stream>>>(plan->d_layers, plan->d_tasks, plan->d_partials);
  RIGL_LAUNCH_CHECK("k_train_summary");
  k_train_summary_finalize<<<plan->n_params, kSgdThreads, 0, stream>>>(plan->d_layers, plan->d_partials, out_dev);
  RIGL_LAUNCH_CHECK("k_train_summary_finalize");
  return RIGL_OK;
}
