// KT: the residual tail of PnP's feature-injected ResNet (utils/pnp_utils.py:146-162):
//   hidden_states[n:2n] = hidden_states[:n]; hidden_states[2n:3n] = hidden_states[:n]   (while injecting)
//   out = (shortcut + hidden_states) / output_scale_factor
// in one HBM pass.  The batch is num_inputs segments of n samples, each segment a contiguous run of M = n * E
// elements (E = C * H * W), and injection only changes where a segment reads h: segments 1 and 2 read segment 0.  So
// the kernel streams the segments (blockIdx.y) with 16-byte vectors; the few elements before the first 16-byte boundary
// of a segment and after its last one are done one by one.  A segment whose three pointers sit at different offsets
// from a 16-byte boundary (possible when M % 8 != 0) is streamed element by element.
//
// Rounding follows torch's CUDA half kernels for the reference's two ops: the add is fp16(float(s) + float(h)), and
// `half_tensor / python_float` is computed as fp16(float(sum) * (1.0f / float(osf))) (div_true_kernel_cuda multiplies by
// the reciprocal of a CPU scalar divisor).
#include <cuda_fp16.h>

#include "common.cuh"

namespace vtm {
namespace {

constexpr int TAIL_THREADS = 256;

__device__ __forceinline__ uint4 ld_nc_16(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ void st_16(void* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
               "r"(v.w)
               : "memory");
}

__device__ __forceinline__ float tail_value(float s, float h, float inv) {
  const float sum = __half2float(__float2half_rn(__fadd_rn(s, h)));
  return __fmul_rn(sum, inv);
}

__device__ __forceinline__ __half tail_elem(__half s, __half h, float inv) {
  return __float2half_rn(tail_value(__half2float(s), __half2float(h), inv));
}

__global__ void __launch_bounds__(TAIL_THREADS)
resnet_tail_kernel(const __half* __restrict__ h, const __half* __restrict__ shortcut, __half* __restrict__ out,
                   long long M, int inject, float inv) {
  const int seg = blockIdx.y;
  const long long off = static_cast<long long>(seg) * M;
  const __half* hs = h + ((inject && (seg == 1 || seg == 2)) ? 0 : off);
  const __half* ss = shortcut + off;
  __half* os = out + off;
  const long long tid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long nthreads = static_cast<long long>(gridDim.x) * blockDim.x;
  // elements before the output's first 16-byte boundary (pointers are 2-byte aligned)
  long long head = ((16 - (reinterpret_cast<uintptr_t>(os) & 15)) & 15) >> 1;
  if (head > M) head = M;
  const bool vec = ((reinterpret_cast<uintptr_t>(ss + head) | reinterpret_cast<uintptr_t>(hs + head)) & 15) == 0;
  if (!vec) {
    for (long long i = tid; i < M; i += nthreads) os[i] = tail_elem(ss[i], hs[i], inv);
    return;
  }
  const long long nv = (M - head) >> 3;
  const long long tail0 = head + (nv << 3);
  if (tid < head) os[tid] = tail_elem(ss[tid], hs[tid], inv);
  if (tid < M - tail0) os[tail0 + tid] = tail_elem(ss[tail0 + tid], hs[tail0 + tid], inv);
  const __half* sv = ss + head;
  const __half* hv = hs + head;
  __half* ov = os + head;
  for (long long v = tid; v < nv; v += nthreads) {
    uint4 a = ld_nc_16(sv + (v << 3));
    const uint4 b = ld_nc_16(hv + (v << 3));
    __half2* a2 = reinterpret_cast<__half2*>(&a);
    const __half2* b2 = reinterpret_cast<const __half2*>(&b);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 x = __half22float2(a2[e]), y = __half22float2(b2[e]);
      a2[e] = __floats2half2_rn(tail_value(x.x, y.x, inv), tail_value(x.y, y.y, inv));
    }
    st_16(ov + (v << 3), a);
  }
}

}  // namespace
}  // namespace vtm

extern "C" int vtm_resnet_tail_f16(const void* h_dev, const void* shortcut_dev, void* out_dev, int32_t n,
                                   int32_t num_inputs, int64_t sample_elems, float output_scale_factor, int32_t inject,
                                   void* stream_) {
  using namespace vtm;
  if (!h_dev || !shortcut_dev || !out_dev) return VTM_E_NULL;
  if (n <= 0 || num_inputs <= 0 || sample_elems <= 0) return VTM_E_SHAPE;
  if (num_inputs > 3 || (inject != 0 && inject != 1)) return VTM_E_UNSUPPORTED;
  if (!isfinite(output_scale_factor) || output_scale_factor == 0.f) return VTM_E_UNSUPPORTED;
  if (((reinterpret_cast<uintptr_t>(h_dev) | reinterpret_cast<uintptr_t>(shortcut_dev) |
        reinterpret_cast<uintptr_t>(out_dev)) & 1) != 0)
    return VTM_E_SHAPE;                                             // fp16 tensors are 2-byte aligned
  if (sample_elems > (INT64_MAX / 3) / n) return VTM_E_SHAPE;
  const long long M = static_cast<long long>(n) * sample_elems;
  int sms = 0;
  int rc = cached_sm_count(&sms);
  if (rc) return rc;
  const long long vecs = (M + 7) / 8;
  long long blocks = (vecs + TAIL_THREADS - 1) / TAIL_THREADS;
  const long long cap = (static_cast<long long>(sms) * (2048 / TAIL_THREADS) + num_inputs - 1) / num_inputs;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  const float inv = 1.0f / output_scale_factor;
  resnet_tail_kernel<<<dim3(static_cast<unsigned>(blocks), static_cast<unsigned>(num_inputs)), TAIL_THREADS, 0,
                       static_cast<cudaStream_t>(stream_)>>>(static_cast<const __half*>(h_dev),
                                                             static_cast<const __half*>(shortcut_dev),
                                                             static_cast<__half*>(out_dev), M, inject, inv);
  return launch_rc();
}
