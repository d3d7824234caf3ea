// KI: one DDIM step in place, x <- c * ((x - a * eps) * r) + d * eps with r = 1 / b, its coefficients read on the device.
//   inversion (invert.py:182-211, inversion=True):   a = sigma_prev, b = mu_prev, c = mu, d = sigma
//   sampling  (generate.py:281-311):                 a = sigma,      b = mu,      c = mu_prev, d = sigma_prev
// The coefficients (a, r, c, d) of every step sit in a small device table, and the step is a device-resident counter,
// so a captured CUDA graph that launches this kernel serves every step: its baked-in arguments never change.  When the
// step's trajectory slot is >= 0 the new x is also stored into traj[slot] in the same pass.
//
// Rounding follows torch's CUDA half kernels for the reference's five ops on python-float coefficients: every product
// and sum is computed in fp32 from the fp16 operands and rounded to fp16, and `half / python_float` is a multiplication
// by the reciprocal (div_true_kernel_cuda), which torch takes in double and rounds once to fp32: r = float(1.0 / b), not
// 1.0f / float(b), so the table holds r as the caller computed it.  Explicit _rn intrinsics keep nvcc from fusing a
// product and a sum into one FMA, which would round once instead of twice.
//
// The pass streams 16-byte vectors; the elements before x's first 16-byte boundary and after its last one are done one
// by one, and when eps or the trajectory slot sits at another offset from a 16-byte boundary (possible when n % 8 != 0)
// the whole pass is element by element.
//
// KS (vtm_cfg_ddim_update_f16) is KI's sampling sibling: it takes a chunk's raw UNet output, forms the classifier-free
// guidance combine in the same pass (three more fp16 roundings, generate.py:274-279) and writes x_{t-1} (generate.py:
// 281-311) to `out`, which may be x itself.  No trajectory; the same vectors, head, tail and fallback as KI.
#include <cuda_fp16.h>

#include "common.cuh"

namespace vtm {
namespace {

constexpr int DDIM_THREADS = 256;

struct DdimCoef {
  float a, r, c, d;   // r = 1 / b
};

__device__ __forceinline__ float rh(float v) { return __half2float(__float2half_rn(v)); }

__device__ __forceinline__ float ddim_value(float x, float e, const DdimCoef& k) {
  const float ae = rh(__fmul_rn(e, k.a));        // a * eps
  const float diff = rh(__fsub_rn(x, ae));       // x - a * eps
  const float x0 = rh(__fmul_rn(diff, k.r));     // / b, as * (1 / b)
  const float cx = rh(__fmul_rn(x0, k.c));       // c * pred_x0
  const float de = rh(__fmul_rn(e, k.d));        // d * eps
  return __fadd_rn(cx, de);
}

__device__ __forceinline__ void ddim_elem(__half* x, const __half* eps, __half* tr, long long i, const DdimCoef& k) {
  const __half v = __float2half_rn(ddim_value(__half2float(x[i]), __half2float(eps[i]), k));
  x[i] = v;
  if (tr) tr[i] = v;
}

__device__ __forceinline__ uint4 ld_nc_16(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}

__global__ void __launch_bounds__(DDIM_THREADS)
ddim_update_kernel(__half* __restrict__ x, const __half* __restrict__ eps, long long n, const float* __restrict__ coef,
                   const int32_t* __restrict__ slot_tab, const int32_t* __restrict__ step_dev, int32_t n_steps,
                   __half* __restrict__ traj, int32_t n_slots) {
  const int step = *step_dev;
  if (step < 0 || step >= n_steps) return;
  const float4 raw = reinterpret_cast<const float4*>(coef)[step];
  const DdimCoef k{raw.x, raw.y, raw.z, raw.w};
  const int slot = slot_tab ? slot_tab[step] : -1;
  __half* tr = (slot >= 0 && slot < n_slots) ? traj + static_cast<long long>(slot) * n : nullptr;

  const long long tid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long nthreads = static_cast<long long>(gridDim.x) * blockDim.x;
  // elements before x's first 16-byte boundary (pointers are 2-byte aligned)
  long long head = ((16 - (reinterpret_cast<uintptr_t>(x) & 15)) & 15) >> 1;
  if (head > n) head = n;
  const uintptr_t others = reinterpret_cast<uintptr_t>(eps + head) | (tr ? reinterpret_cast<uintptr_t>(tr + head) : 0);
  if ((others & 15) != 0) {
    for (long long i = tid; i < n; i += nthreads) ddim_elem(x, eps, tr, i, k);
    return;
  }
  const long long nv = (n - head) >> 3;
  const long long tail0 = head + (nv << 3);
  if (tid < head) ddim_elem(x, eps, tr, tid, k);
  if (tid < n - tail0) ddim_elem(x, eps, tr, tail0 + tid, k);
  uint4* xv = reinterpret_cast<uint4*>(x + head);
  const __half* ev = eps + head;
  uint4* tv = tr ? reinterpret_cast<uint4*>(tr + head) : nullptr;
  for (long long v = tid; v < nv; v += nthreads) {
    uint4 a = xv[v];
    const uint4 b = ld_nc_16(ev + (v << 3));
    __half2* a2 = reinterpret_cast<__half2*>(&a);
    const __half2* b2 = reinterpret_cast<const __half2*>(&b);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 p = __half22float2(a2[e]), q = __half22float2(b2[e]);
      a2[e] = __floats2half2_rn(ddim_value(p.x, q.x, k), ddim_value(p.y, q.y, k));
    }
    xv[v] = a;
    if (tv) tv[v] = a;
  }
}

// KS: the sampling step's guidance combine and DDIM update, out <- c * ((x - a * e) * r) + d * e with
//   e = u + g * (c_eps - u)                         generate.py:274-279 (noise_pred_uncond, noise_pred_cond)
//   a = sigma, r = 1 / mu, c = mu_prev, d = sigma_prev   generate.py:281-311 (inversion=False)
// u and c_eps are the last two of the `samples` blocks of the UNet output.  The three guidance ops round to fp16 as
// torch's half sub / mul / add do; g is float(guidance), the opmath value torch takes a python scalar at.
__device__ __forceinline__ float cfg_ddim_value(float x, float u, float c, float g, const DdimCoef& k) {
  const float diff = rh(__fsub_rn(c, u));        // cond - uncond
  const float gd = rh(__fmul_rn(g, diff));       // guidance * (cond - uncond)
  const float e = rh(__fadd_rn(u, gd));          // uncond + ...
  return ddim_value(x, e, k);
}

__device__ __forceinline__ void cfg_ddim_elem(const __half* x, const __half* u, const __half* c, __half* out,
                                              long long i, float g, const DdimCoef& k) {
  out[i] = __float2half_rn(cfg_ddim_value(__half2float(x[i]), __half2float(u[i]), __half2float(c[i]), g, k));
}

// x and out may be the same buffer (every element is read by the thread that writes it), so neither is __restrict__
// and x is not read through the non-coherent path.
__global__ void __launch_bounds__(DDIM_THREADS)
cfg_ddim_update_kernel(const __half* x, const __half* __restrict__ u, const __half* __restrict__ c, long long n,
                       float g, const float* __restrict__ coef, const int32_t* __restrict__ step_dev, int32_t n_steps,
                       __half* out) {
  const int step = *step_dev;
  if (step < 0 || step >= n_steps) return;
  const float4 raw = reinterpret_cast<const float4*>(coef)[step];
  const DdimCoef k{raw.x, raw.y, raw.z, raw.w};

  const long long tid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long nthreads = static_cast<long long>(gridDim.x) * blockDim.x;
  // elements before out's first 16-byte boundary (pointers are 2-byte aligned)
  long long head = ((16 - (reinterpret_cast<uintptr_t>(out) & 15)) & 15) >> 1;
  if (head > n) head = n;
  const uintptr_t others = reinterpret_cast<uintptr_t>(x + head) | reinterpret_cast<uintptr_t>(u + head) |
                           reinterpret_cast<uintptr_t>(c + head);
  if ((others & 15) != 0) {
    for (long long i = tid; i < n; i += nthreads) cfg_ddim_elem(x, u, c, out, i, g, k);
    return;
  }
  const long long nv = (n - head) >> 3;
  const long long tail0 = head + (nv << 3);
  if (tid < head) cfg_ddim_elem(x, u, c, out, tid, g, k);
  if (tid < n - tail0) cfg_ddim_elem(x, u, c, out, tail0 + tid, g, k);
  const uint4* xv = reinterpret_cast<const uint4*>(x + head);
  const __half* uv = u + head;
  const __half* cv = c + head;
  uint4* ov = reinterpret_cast<uint4*>(out + head);
  for (long long v = tid; v < nv; v += nthreads) {
    uint4 a = xv[v];
    const uint4 p = ld_nc_16(uv + (v << 3));
    const uint4 q = ld_nc_16(cv + (v << 3));
    __half2* a2 = reinterpret_cast<__half2*>(&a);
    const __half2* p2 = reinterpret_cast<const __half2*>(&p);
    const __half2* q2 = reinterpret_cast<const __half2*>(&q);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 xf = __half22float2(a2[e]), uf = __half22float2(p2[e]), cf = __half22float2(q2[e]);
      a2[e] = __floats2half2_rn(cfg_ddim_value(xf.x, uf.x, cf.x, g, k), cfg_ddim_value(xf.y, uf.y, cf.y, g, k));
    }
    ov[v] = a;
  }
}

bool overlaps(const void* a, long long a_bytes, const void* b, long long b_bytes) {
  const uintptr_t pa = reinterpret_cast<uintptr_t>(a), pb = reinterpret_cast<uintptr_t>(b);
  return pa < pb + static_cast<uintptr_t>(b_bytes) && pb < pa + static_cast<uintptr_t>(a_bytes);
}

unsigned ddim_blocks(long long n, int sms) {
  long long blocks = (n + 8LL * DDIM_THREADS - 1) / (8LL * DDIM_THREADS);
  const long long cap = static_cast<long long>(sms) * (2048 / DDIM_THREADS);
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return static_cast<unsigned>(blocks);
}

}  // namespace
}  // namespace vtm

extern "C" int vtm_cfg_ddim_update_f16(const void* x_dev, const void* eps_dev, int64_t n, int32_t samples,
                                       float guidance, const float* coef_dev, const int32_t* step_dev, int32_t n_steps,
                                       void* out_dev, void* stream_) {
  using namespace vtm;
  if (!x_dev || !eps_dev || !coef_dev || !step_dev || !out_dev) return VTM_E_NULL;
  if (n <= 0 || n_steps <= 0 || (samples != 2 && samples != 3) || n > INT64_MAX / 2 / samples) return VTM_E_SHAPE;
  if (((reinterpret_cast<uintptr_t>(x_dev) | reinterpret_cast<uintptr_t>(eps_dev) |
        reinterpret_cast<uintptr_t>(out_dev)) & 1) != 0)
    return VTM_E_SHAPE;                                             // fp16 tensors are 2-byte aligned
  if ((reinterpret_cast<uintptr_t>(coef_dev) & 15) != 0 || (reinterpret_cast<uintptr_t>(step_dev) & 3) != 0)
    return VTM_E_SHAPE;                                             // the table is read as one float4 per step
  const long long bytes = 2LL * n;
  if ((out_dev != x_dev && overlaps(out_dev, bytes, x_dev, bytes)) || overlaps(out_dev, bytes, eps_dev, samples * bytes))
    return VTM_E_SHAPE;                                             // out is x itself or apart from x and eps
  int sms = 0;
  int rc = cached_sm_count(&sms);
  if (rc) return rc;
  const __half* eps = static_cast<const __half*>(eps_dev);
  cfg_ddim_update_kernel<<<ddim_blocks(n, sms), DDIM_THREADS, 0, static_cast<cudaStream_t>(stream_)>>>(
      static_cast<const __half*>(x_dev), eps + (samples - 2) * n, eps + (samples - 1) * n, n, guidance, coef_dev,
      step_dev, n_steps, static_cast<__half*>(out_dev));
  return launch_rc();
}

extern "C" int vtm_ddim_update_f16(void* x_dev, const void* eps_dev, int64_t n, const float* coef_dev,
                                   const int32_t* slot_dev, const int32_t* step_dev, int32_t n_steps, void* traj_dev,
                                   int32_t n_slots, void* stream_) {
  using namespace vtm;
  if (!x_dev || !eps_dev || !coef_dev || !step_dev) return VTM_E_NULL;
  if (slot_dev && !traj_dev) return VTM_E_NULL;
  if (n <= 0 || n_steps <= 0 || n_slots < 0 || (slot_dev && n_slots == 0)) return VTM_E_SHAPE;
  if (((reinterpret_cast<uintptr_t>(x_dev) | reinterpret_cast<uintptr_t>(eps_dev) |
        reinterpret_cast<uintptr_t>(traj_dev)) & 1) != 0)
    return VTM_E_SHAPE;                                             // fp16 tensors are 2-byte aligned
  if ((reinterpret_cast<uintptr_t>(coef_dev) & 15) != 0 || (reinterpret_cast<uintptr_t>(step_dev) & 3) != 0 ||
      (reinterpret_cast<uintptr_t>(slot_dev) & 3) != 0)
    return VTM_E_SHAPE;                                             // the table is read as one float4 per step
  if (n_slots > 0 && n > INT64_MAX / n_slots) return VTM_E_SHAPE;
  int sms = 0;
  int rc = cached_sm_count(&sms);
  if (rc) return rc;
  long long blocks = (n + 8LL * DDIM_THREADS - 1) / (8LL * DDIM_THREADS);
  const long long cap = static_cast<long long>(sms) * (2048 / DDIM_THREADS);
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  ddim_update_kernel<<<static_cast<unsigned>(blocks), DDIM_THREADS, 0, static_cast<cudaStream_t>(stream_)>>>(
      static_cast<__half*>(x_dev), static_cast<const __half*>(eps_dev), n, coef_dev, slot_dev, step_dev, n_steps,
      static_cast<__half*>(traj_dev), n_slots);
  return launch_rc();
}
