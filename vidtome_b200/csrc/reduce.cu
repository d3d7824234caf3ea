// Merge with a reduction — the non-"replace" modes of the merge closure (vidtome/merge.py:126-131):
//   dst = dst.scatter_reduce(-2, dst_idx, src[src_idx], reduce=mode, include_self=True);  out = cat([unm, dst])
// for mode in {mean, sum, amax, amin}.  No caller in the reference passes a mode (SURVEY §0.3), so this is an
// operator-API feature, not part of the composed per-block plan (a reduction is not a row gather: levels do not
// compose into one map).
//
// Sums are order-independent and exact: every fp16 value is an integer multiple of 2^-24 below 2^16, so a row of
// int64 fixed-point accumulators (value * 2^24) holds the exact sum of up to 2^22 tokens, and 64-bit integer atomics
// make the result independent of the order in which src rows arrive.  The reference accumulates in fp16 in index
// order on the CPU and with fp16 atomics in arbitrary order on CUDA; both agree with the exact sum whenever the
// partial sums are representable (the "exact" fixtures), and differ from it by fp16 rounding otherwise.
// mean = fp16(float(sum) / float(count)), as torch divides the fp16 sum by the count in fp32.
// amax / amin use the same accumulators with an order-preserving integer image of the fp16 value.
// Inputs must be finite.
#include <cuda_fp16.h>

#include "common.cuh"
#include "ptx.cuh"

namespace vtm {
namespace {

enum { MODE_MEAN = 1, MODE_SUM = 2, MODE_AMAX = 3, MODE_AMIN = 4 };

__device__ __forceinline__ long long to_acc(__half h, int mode) {
  if (mode <= MODE_SUM) return __float2ll_rn(__half2float(h) * 16777216.f);   // exact: 11-bit significand * 2^24
  uint32_t u = __half_as_ushort(h);
  if (u == 0x8000u) u = 0;                                                    // -0 == +0
  return (u & 0x8000u) ? -static_cast<long long>(u & 0x7FFFu) : static_cast<long long>(u);
}
__device__ __forceinline__ __half from_acc(long long a, int cnt, int mode) {
  if (mode == MODE_SUM) return __double2half(static_cast<double>(a) * (1.0 / 16777216.0));
  if (mode == MODE_MEAN) {
    const float s = static_cast<float>(static_cast<double>(a) * (1.0 / 16777216.0));
    return __float2half_rn(s / static_cast<float>(cnt));
  }
  const uint32_t u = a < 0 ? (0x8000u | static_cast<uint32_t>(-a)) : static_cast<uint32_t>(a);
  return __ushort_as_half(static_cast<unsigned short>(u));
}

// one warp per row; lanes stride over 8-element vectors
__global__ void __launch_bounds__(256)
reduce_init_kernel(const __half* __restrict__ x, long long x_bs, Split sp, int r, int Bp, const int* __restrict__ edge,
                   int B, int C, int mode, __half* __restrict__ y, long long* __restrict__ acc, int* __restrict__ cnt) {
  resolve_split(sp);
  const int unm = sp.Ns - r, Lout = unm + sp.Nd;
  const long long warp = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= static_cast<long long>(B) * Lout) return;
  const int b = static_cast<int>(warp / Lout), t = static_cast<int>(warp % Lout);
  const int bp = Bp == 1 ? 0 : b;
  if (t < unm) {   // unmerged src rows, in edge order (merge.py:124)
    const int pos = src_pos(sp, edge[static_cast<long long>(bp) * sp.Ns + r + t]);
    const uint4* s = reinterpret_cast<const uint4*>(x + b * x_bs + static_cast<long long>(pos) * C);
    uint4* d = reinterpret_cast<uint4*>(y + (static_cast<long long>(b) * Lout + t) * C);
    for (int v = lane; v < C / 8; v += 32) d[v] = s[v];
  } else {         // dst rows seed the accumulators (include_self=True)
    const int j = t - unm;
    const __half* s = x + b * x_bs + static_cast<long long>(dst_pos(sp, j)) * C;
    long long* a = acc + (static_cast<long long>(b) * sp.Nd + j) * C;
    for (int c = lane; c < C; c += 32) a[c] = to_acc(s[c], mode);
    if (lane == 0) cnt[static_cast<long long>(b) * sp.Nd + j] = 1;
  }
}

__global__ void __launch_bounds__(256)
reduce_scatter_kernel(const __half* __restrict__ x, long long x_bs, Split sp, int r, int Bp,
                      const unsigned long long* __restrict__ keys, const int* __restrict__ edge, int B, int C, int mode,
                      long long* __restrict__ acc, int* __restrict__ cnt) {
  resolve_split(sp);
  const long long warp = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= static_cast<long long>(B) * r) return;
  const int b = static_cast<int>(warp / r), k = static_cast<int>(warp % r);
  const int bp = Bp == 1 ? 0 : b;
  const int i = edge[static_cast<long long>(bp) * sp.Ns + k];                       // src_idx[k]   (merge.py:101,116)
  const uint32_t arg = 0xFFFFFFFFu - static_cast<uint32_t>(keys[static_cast<long long>(bp) * sp.Ns + i] & 0xFFFFFFFFull);
  const int j = static_cast<int>(arg % static_cast<uint32_t>(sp.Nd));              // dst_idx[k]   (merge.py:102-103,117)
  const __half* s = x + b * x_bs + static_cast<long long>(src_pos(sp, i)) * C;
  unsigned long long* a = reinterpret_cast<unsigned long long*>(acc + (static_cast<long long>(b) * sp.Nd + j) * C);
  for (int c = lane; c < C; c += 32) {
    const long long v = to_acc(s[c], mode);
    if (mode <= MODE_SUM) atomicAdd(a + c, static_cast<unsigned long long>(v));     // two's complement: signed add
    else if (mode == MODE_AMAX) atomicMax(reinterpret_cast<long long*>(a) + c, v);
    else atomicMin(reinterpret_cast<long long*>(a) + c, v);
  }
  if (lane == 0 && mode == MODE_MEAN) atomicAdd(cnt + static_cast<long long>(b) * sp.Nd + j, 1);
}

__global__ void __launch_bounds__(256)
reduce_final_kernel(Split sp, int r, int B, int C, int mode, const long long* __restrict__ acc,
                    const int* __restrict__ cnt, __half* __restrict__ y) {
  const int unm = sp.Ns - r, Lout = unm + sp.Nd;
  const long long total = static_cast<long long>(B) * sp.Nd * C;
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long row = e / C;
    const int c = static_cast<int>(e - row * C);
    const int b = static_cast<int>(row / sp.Nd), j = static_cast<int>(row % sp.Nd);
    y[(static_cast<long long>(b) * Lout + unm + j) * C + c] = from_acc(acc[e], cnt[row], mode);
  }
}

size_t align256(size_t v) { return (v + 255) & ~static_cast<size_t>(255); }

}  // namespace
}  // namespace vtm

extern "C" size_t vtm_merge_reduce_workspace_bytes(int32_t B, int32_t Nd, int32_t C) {
  if (B <= 0 || Nd <= 0 || C <= 0) return 0;
  return vtm::align256(sizeof(long long) * static_cast<size_t>(B) * Nd * C) + vtm::align256(sizeof(int) * static_cast<size_t>(B) * Nd);
}

extern "C" int vtm_merge_reduce(const void* x_dev, int64_t x_batch_stride, const vtm_split_t* split, int32_t r,
                                int32_t Bp, const uint64_t* keys_dev, const int32_t* edge_dev, int32_t B, int32_t C,
                                int32_t mode, void* y_dev, void* ws_dev, size_t ws_bytes, void* stream_) {
  using namespace vtm;
  Split sp;
  int rc = make_split(split, &sp);
  if (rc) return rc;
  if (sp.glob_len_dev) return VTM_E_SPLIT;   // device counts: only the replace-mode row gathers have that path
  if (!x_dev || !y_dev || !ws_dev) return VTM_E_NULL;
  if (sp.Ns > 0 && (!keys_dev || !edge_dev)) return VTM_E_NULL;
  if (B <= 0 || C <= 0 || (C % 8) != 0 || r < 0 || r > sp.Ns || sp.Nd <= 0 || (Bp != 1 && Bp != B)) return VTM_E_SHAPE;
  if (mode < MODE_MEAN || mode > MODE_AMIN) return VTM_E_UNSUPPORTED;
  if (ws_bytes < vtm_merge_reduce_workspace_bytes(B, sp.Nd, C)) return VTM_E_WS;
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  long long* acc = static_cast<long long*>(ws_dev);
  int* cnt = reinterpret_cast<int*>(static_cast<char*>(ws_dev) + align256(sizeof(long long) * static_cast<size_t>(B) * sp.Nd * C));
  const int Lout = sp.Ns - r + sp.Nd;
  const long long w1 = static_cast<long long>(B) * Lout;
  reduce_init_kernel<<<static_cast<unsigned>((w1 * 32 + 255) / 256), 256, 0, st>>>(
      static_cast<const __half*>(x_dev), x_batch_stride, sp, r, Bp, edge_dev, B, C, mode, static_cast<__half*>(y_dev), acc, cnt);
  rc = launch_rc();
  if (rc) return rc;
  if (r > 0) {
    const long long w2 = static_cast<long long>(B) * r;
    reduce_scatter_kernel<<<static_cast<unsigned>((w2 * 32 + 255) / 256), 256, 0, st>>>(
        static_cast<const __half*>(x_dev), x_batch_stride, sp, r, Bp, reinterpret_cast<const unsigned long long*>(keys_dev),
        edge_dev, B, C, mode, acc, cnt);
    rc = launch_rc();
    if (rc) return rc;
  }
  const long long total = static_cast<long long>(B) * sp.Nd * C;
  long long blocks = (total + 255) / 256;
  int sms = 0;
  rc = cached_sm_count(&sms);
  if (rc) return rc;
  if (blocks > static_cast<long long>(sms) * 16) blocks = static_cast<long long>(sms) * 16;
  reduce_final_kernel<<<static_cast<unsigned>(blocks), 256, 0, st>>>(sp, r, B, C, mode, acc, cnt, static_cast<__half*>(y_dev));
  return launch_rc();
}
