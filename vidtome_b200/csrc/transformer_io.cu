// Entry of diffusers' Transformer2DModel.forward on NCHW activations: GroupNorm(groups, C) whose output is written
// straight as token-major rows [n, HW, C], the layout every other kernel of the library reads (DESIGN §3).  Replaces
//   x = norm(x); ...; x = x.permute(0, 2, 3, 1).reshape(n, h * w, C)
// of Transformer2DModel.forward (third-party code; its arithmetic is torch's, not pinned by the reference, like attn1's:
// SURVEY §8c).  Two kernels, because a group's statistics need the whole group before its first element can be
// normalised:
//   KG1  vtm_group_norm_stats_f16   one read of x   -> (mean, rstd) per (sample, group)
//   KG2  vtm_group_norm_tokens_f16  one read of x   -> one write of y, transposed through shared memory
// The exit of the wrapper (proj_out + residual back to NCHW) is the NchwEpi epilogue of the projection GEMM (linear.cu).
#include <cuda_fp16.h>

#include "common.cuh"
#include "ptx.cuh"

namespace vtm {
namespace {

// ---------------------------------------------------------------------------------------------------------------------
// KG1.  A (sample, group) is one contiguous run of R = (C / groups) * HW halfs starting at run * R.
//
// Arithmetic (all fp32).  A thread reduces each 16-byte vector of eight halfs to (8, m, M2) with m = (sum of the eight)
// / 8 and M2 = sum (v - m)^2, two passes over registers, and folds it into its running (n, mean, M2) with the pairwise
// update of Chan, Golub and LeVeque:
//     n = na + nb;  d = mb - ma;  w = nb / n;  mean = ma + d w;  M2 = Ma + Mb + d^2 na w.
// Threads, warps and (for a split run) CTAs are combined by the same update.  No term is ever a difference of two
// large sums, so a mean that is large against the spread (mean 1000, spread 1/8) costs no digits: every M2 is a sum of
// squared deviations from a mean taken over the same elements.  The combination order is fixed by the shape alone, so
// the result is the same on every call (CUDA-graph replays included).
//
// Grid.  Runs of at most SMALL_RUN halfs take one warp each, eight per CTA: grid = ceil(runs / 8).  Longer runs take one
// 256-thread CTA per piece, a run being cut into S pieces when there are too few runs to fill the machine:
//     S = 1                                          if runs >= FILL_CTAS or R <= PIECE
//     S = min(ceil(R / PIECE), ceil(FILL_CTAS / runs))  otherwise
// (PIECE = 8192 halfs, FILL_CTAS = 512: about four CTAs per SM of an H100).  C = 320, HW = 4096, 32 items: 1024 runs of
// 40960 halfs, S = 1, 1024 CTAs.  One 768 x 768 latent (HW = 9216, C = 320): 32 runs of 92160 halfs, S = 12, 384 CTAs.
// With S > 1 the pieces' (n, mean, M2) go to the workspace and a second, tiny kernel combines them in piece order.
constexpr int SMALL_RUN = 2048;
constexpr int PIECE = 8192;
constexpr int FILL_CTAS = 512;
constexpr int STATS_THREADS = 256;

struct Moments {
  float n, mean, m2;
};

// (a) <- (a) U (b); b may be empty
__device__ __forceinline__ void chan(Moments& a, const Moments& b) {
  if (b.n == 0.f) return;
  const float n = __fadd_rn(a.n, b.n);
  const float d = __fsub_rn(b.mean, a.mean);
  const float w = __fdiv_rn(b.n, n);
  const float dw = __fmul_rn(d, w);
  a.mean = __fadd_rn(a.mean, dw);
  a.m2 = __fadd_rn(__fadd_rn(a.m2, b.m2), __fmul_rn(__fmul_rn(d, dw), a.n));
  a.n = n;
}

__device__ __forceinline__ Moments moments8(const uint4& v) {
  const __half2* h = reinterpret_cast<const __half2*>(&v);
  float f[8];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float2 t = __half22float2(h[e]);
    f[2 * e] = t.x;
    f[2 * e + 1] = t.y;
  }
  const float s = __fadd_rn(__fadd_rn(__fadd_rn(f[0], f[1]), __fadd_rn(f[2], f[3])),
                            __fadd_rn(__fadd_rn(f[4], f[5]), __fadd_rn(f[6], f[7])));
  Moments m;
  m.n = 8.f;
  m.mean = __fmul_rn(s, 0.125f);
  float q = 0.f;
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const float d = __fsub_rn(f[e], m.mean);
    q = __fmaf_rn(d, d, q);
  }
  m.m2 = q;
  return m;
}

// This thread's share of the halfs [p, p + len): the elements before the first and after the last 16-byte boundary are
// read one at a time (one per thread), the vectors in between round-robin over the nthreads threads.
__device__ __forceinline__ Moments piece_moments(const __half* p, long long len, int tid, int nthreads) {
  Moments acc{0.f, 0.f, 0.f};
  const uintptr_t addr = reinterpret_cast<uintptr_t>(p);
  long long head = static_cast<long long>(((16 - (addr & 15)) & 15) >> 1);
  if (head > len) head = len;
  const long long nvec = (len - head) >> 3;
  const long long tail0 = head + (nvec << 3);
  if (tid < head) acc = Moments{1.f, __half2float(p[tid]), 0.f};
  const uint4* v = reinterpret_cast<const uint4*>(p + head);
  long long i = tid;
  for (; i + 3LL * nthreads < nvec; i += 4LL * nthreads) {       // four loads in flight per thread
    const uint4 a = __ldg(v + i), b = __ldg(v + i + nthreads), c = __ldg(v + i + 2LL * nthreads),
                d = __ldg(v + i + 3LL * nthreads);
    chan(acc, moments8(a));
    chan(acc, moments8(b));
    chan(acc, moments8(c));
    chan(acc, moments8(d));
  }
  for (; i < nvec; i += nthreads) chan(acc, moments8(__ldg(v + i)));
  if (tail0 + tid < len) chan(acc, Moments{1.f, __half2float(p[tail0 + tid]), 0.f});
  return acc;
}

__device__ __forceinline__ Moments warp_moments(Moments m) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    Moments b;
    b.n = __shfl_xor_sync(0xffffffffu, m.n, o);
    b.mean = __shfl_xor_sync(0xffffffffu, m.mean, o);
    b.m2 = __shfl_xor_sync(0xffffffffu, m.m2, o);
    // both partners must fold in the same order to hold the same value afterwards: lower lane's set first
    if (threadIdx.x & o) {
      Moments a = b;
      chan(a, m);
      m = a;
    } else {
      chan(m, b);
    }
  }
  return m;
}

__device__ __forceinline__ void store_stats(float* stats, long long run, const Moments& m, float eps) {
  const float var = __fdiv_rn(m.m2, m.n);                                     // biased, as torch's group_norm
  stats[2 * run] = m.mean;
  stats[2 * run + 1] = __fdiv_rn(1.f, __fsqrt_rn(__fadd_rn(var, eps)));
}

// one warp per run
__global__ void __launch_bounds__(STATS_THREADS)
group_norm_stats_small_kernel(const __half* __restrict__ x, long long runs, int R, float eps, float* __restrict__ stats) {
  const long long run = static_cast<long long>(blockIdx.x) * (STATS_THREADS / 32) + (threadIdx.x >> 5);
  if (run >= runs) return;
  const Moments m = warp_moments(piece_moments(x + run * R, R, threadIdx.x & 31, 32));
  if ((threadIdx.x & 31) == 0) store_stats(stats, run, m, eps);
}

// one CTA per (run, piece); S == 1 writes the statistics, S > 1 the piece's moments [runs, S, 3]
__global__ void __launch_bounds__(STATS_THREADS)
group_norm_stats_large_kernel(const __half* __restrict__ x, long long R, int S, long long piece, float eps,
                              float* __restrict__ stats, float* __restrict__ partial) {
  __shared__ Moments warp_m[STATS_THREADS / 32];
  const long long run = blockIdx.x / S;
  const int s = blockIdx.x - static_cast<int>(run) * S;
  const long long lo = s * piece;
  long long len = R - lo;
  if (len > piece) len = piece;
  const Moments m = warp_moments(piece_moments(x + run * R + lo, len, threadIdx.x, STATS_THREADS));
  if ((threadIdx.x & 31) == 0) warp_m[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    Moments a = warp_m[0];
#pragma unroll
    for (int w = 1; w < STATS_THREADS / 32; ++w) chan(a, warp_m[w]);
    if (S == 1) {
      store_stats(stats, run, a, eps);
    } else {
      float* o = partial + (run * S + s) * 3;
      o[0] = a.n; o[1] = a.mean; o[2] = a.m2;
    }
  }
}

__global__ void group_norm_stats_combine_kernel(const float* __restrict__ partial, long long runs, int S, float eps,
                                                float* __restrict__ stats) {
  const long long run = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (run >= runs) return;
  const float* p = partial + run * S * 3;
  Moments a{p[0], p[1], p[2]};
  for (int s = 1; s < S; ++s) chan(a, Moments{p[3 * s], p[3 * s + 1], p[3 * s + 2]});
  store_stats(stats, run, a, eps);
}

// pieces per run (see "Grid" above)
int stats_split(long long runs, long long R) {
  if (R <= SMALL_RUN || runs >= FILL_CTAS || R <= PIECE) return 1;
  const long long by_len = (R + PIECE - 1) / PIECE, by_fill = (FILL_CTAS + runs - 1) / runs;
  return static_cast<int>(by_len < by_fill ? by_len : by_fill);
}

// ---------------------------------------------------------------------------------------------------------------------
// KG2.  y[i, p, c] = fp16(fma((float(x[i, c, p]) - mean) * rstd, gamma[c], beta[c])), mean and rstd those of c's group:
// an fp32 subtraction, an fp32 multiplication and one fma, each rounded to nearest, in this order (torch's kernel
// folds rstd * gamma and mean into two per-channel constants first; the two agree to an fp16 ulp).
//
// One CTA transposes a tile of 64 tokens x 64 channels: grid = (ceil(HW / 64), ceil(C / 64), n), 256 threads.
// Load: a thread takes eight consecutive tokens of one channel (one 16-byte load; eight lanes cover the 128-byte line of
// the tile's 64 tokens) and normalises them.  Lanes l and l ^ 8 hold neighbouring channels of the same tokens; they
// swap halves, so that each ends up with four tokens x (even channel, odd channel) as four 32-bit words.
// Shared tile: T[token][32 words] (64 channels of a token = the 128 bytes that go out as one line), word cw of token p
// stored at cw ^ f(p), f(p) = 4 ((p >> 3) & 7) + 2 ((p >> 2) & 1).  For one store instruction a warp's lanes differ in
// (p >> 3) & 7 (eight values), (p >> 2) & 1 and cw & 1: 32 different banks.  For the read a lane takes the 16-byte
// chunk m of token p, found at chunk m ^ ((p >> 3) & 7) with its two 8-byte halves swapped when (p >> 2) & 1; eight
// lanes read one token's 128 bytes (all 32 banks) and store them as one full line of y.
// Tiles that reach past HW or C, and every tile when HW % 8 != 0 or x is not 16-byte aligned (a channel row then does
// not start on a 16-byte boundary), load element by element with range checks; the rest of the kernel is the same.
constexpr int GT_THREADS = 256;

__global__ void __launch_bounds__(GT_THREADS)
group_norm_tokens_kernel(const __half* __restrict__ x, const float* __restrict__ stats, const __half* __restrict__ gamma,
                         const __half* __restrict__ beta, int C, int HW, int groups, int vec_ok,
                         __half* __restrict__ y) {
  __shared__ __align__(16) uint32_t tile[64 * 32];
  const int p0 = blockIdx.x * 64, c0 = blockIdx.y * 64, i = blockIdx.z;
  const int cpg = C / groups;
  const int lane_odd = (threadIdx.x >> 3) & 1;                  // this thread's channel is the odd one of its pair
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int item = threadIdx.x + GT_THREADS * r;
    const int k = item & 7, cl = item >> 3;                     // token octet, channel within the tile
    const int c = c0 + cl, p = p0 + 8 * k;
    uint4 raw = make_uint4(0, 0, 0, 0);
    float mean = 0.f, rstd = 0.f, g = 0.f, b = 0.f;
    if (c < C) {
      const __half* src = x + (static_cast<long long>(i) * C + c) * HW + p;
      if (vec_ok && p + 8 <= HW) {
        raw = __ldg(reinterpret_cast<const uint4*>(src));
      } else {
        __half* e = reinterpret_cast<__half*>(&raw);
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (p + j < HW) e[j] = src[j];
      }
      const float2 st = __ldg(reinterpret_cast<const float2*>(stats) + static_cast<long long>(i) * groups + c / cpg);
      mean = st.x; rstd = st.y;
      g = gamma ? __half2float(gamma[c]) : 1.f;
      b = beta ? __half2float(beta[c]) : 0.f;
    }
    uint32_t w[4];
    {
      const __half2* h = reinterpret_cast<const __half2*>(&raw);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 t = __half22float2(h[e]);
        w[e] = pack_f16x2(__fmaf_rn(__fmul_rn(__fsub_rn(t.x, mean), rstd), g, b),
                          __fmaf_rn(__fmul_rn(__fsub_rn(t.y, mean), rstd), g, b));
      }
    }
    // the even channel keeps tokens 0-3 and gets its neighbour's, the odd channel keeps 4-7
    const uint32_t s0 = __shfl_xor_sync(0xffffffffu, lane_odd ? w[0] : w[2], 8);
    const uint32_t s1 = __shfl_xor_sync(0xffffffffu, lane_odd ? w[1] : w[3], 8);
    const uint32_t e0 = lane_odd ? s0 : w[0], e1 = lane_odd ? s1 : w[1];      // even channel, two tokens per word
    const uint32_t o0 = lane_odd ? w[2] : s0, o1 = lane_odd ? w[3] : s1;      // odd channel
    const uint32_t out[4] = {__byte_perm(e0, o0, 0x5410), __byte_perm(e0, o0, 0x7632), __byte_perm(e1, o1, 0x5410),
                             __byte_perm(e1, o1, 0x7632)};
    const int cw = cl >> 1;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int pl = 8 * k + 4 * lane_odd + j;
      tile[pl * 32 + (cw ^ (4 * k + 2 * lane_odd))] = out[j];
    }
  }
  __syncthreads();
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int item = threadIdx.x + GT_THREADS * r;
    const int m = item & 7, pl = item >> 3;
    const int p = p0 + pl, c = c0 + 8 * m;
    if (p >= HW || c >= C) continue;
    uint4 v = *reinterpret_cast<const uint4*>(&tile[pl * 32 + 4 * (m ^ ((pl >> 3) & 7))]);
    if ((pl >> 2) & 1) v = make_uint4(v.z, v.w, v.x, v.y);
    *reinterpret_cast<uint4*>(y + (static_cast<long long>(i) * HW + p) * C + c) = v;
  }
}

int norm_args(const void* x_dev, int n, int C, int HW, int groups) {
  if (!x_dev) return VTM_E_NULL;
  if (n <= 0 || C <= 0 || HW <= 0 || groups <= 0 || C % groups != 0) return VTM_E_SHAPE;
  if (reinterpret_cast<uintptr_t>(x_dev) % 2 != 0) return VTM_E_SHAPE;
  return VTM_OK;
}

}  // namespace
}  // namespace vtm

extern "C" size_t vtm_group_norm_stats_workspace_bytes(int32_t n, int32_t C, int32_t HW, int32_t groups) {
  if (n <= 0 || C <= 0 || HW <= 0 || groups <= 0 || C % groups != 0) return 0;
  const long long runs = static_cast<long long>(n) * groups, R = static_cast<long long>(C / groups) * HW;
  const int S = vtm::stats_split(runs, R);
  return S == 1 ? 0 : static_cast<size_t>(runs) * S * 3 * sizeof(float);
}

extern "C" int vtm_group_norm_stats_f16(const void* x_dev, int32_t n, int32_t C, int32_t HW, int32_t groups, float eps,
                                        float* stats_dev, void* ws_dev, size_t ws_bytes, void* stream_) {
  using namespace vtm;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int rc = norm_args(x_dev, n, C, HW, groups);
  if (rc) return rc;
  if (!stats_dev) return VTM_E_NULL;
  if (reinterpret_cast<uintptr_t>(stats_dev) % 8 != 0 || !(eps >= 0.f)) return VTM_E_SHAPE;
  const long long runs = static_cast<long long>(n) * groups, R = static_cast<long long>(C / groups) * HW;
  const __half* x = static_cast<const __half*>(x_dev);
  if (R <= SMALL_RUN) {
    const long long grid = (runs + STATS_THREADS / 32 - 1) / (STATS_THREADS / 32);
    if (grid > 0x7fffffffLL) return VTM_E_SHAPE;
    group_norm_stats_small_kernel<<<static_cast<unsigned>(grid), STATS_THREADS, 0, stream>>>(
        x, runs, static_cast<int>(R), eps, stats_dev);
    return launch_rc();
  }
  const int S = stats_split(runs, R);
  if (runs * S > 0x7fffffffLL) return VTM_E_SHAPE;
  const long long piece = S == 1 ? R : ((R + S - 1) / S + 7) & ~7LL;          // whole 16-byte vectors per piece
  if (S > 1) {
    if (!ws_dev) return VTM_E_NULL;
    if (ws_bytes < static_cast<size_t>(runs) * S * 3 * sizeof(float)) return VTM_E_WS;
    if (reinterpret_cast<uintptr_t>(ws_dev) % 4 != 0) return VTM_E_SHAPE;
  }
  float* partial = static_cast<float*>(ws_dev);
  group_norm_stats_large_kernel<<<static_cast<unsigned>(runs * S), STATS_THREADS, 0, stream>>>(x, R, S, piece, eps,
                                                                                             stats_dev, partial);
  rc = launch_rc();
  if (rc || S == 1) return rc;
  group_norm_stats_combine_kernel<<<static_cast<unsigned>((runs + 127) / 128), 128, 0, stream>>>(partial, runs, S, eps,
                                                                                                  stats_dev);
  return launch_rc();
}

extern "C" int vtm_group_norm_tokens_f16(const void* x_dev, const float* stats_dev, const void* gamma_dev,
                                         const void* beta_dev, int32_t n, int32_t C, int32_t HW, int32_t groups,
                                         void* y_dev, void* stream_) {
  using namespace vtm;
  int rc = norm_args(x_dev, n, C, HW, groups);
  if (rc) return rc;
  if (!stats_dev || !y_dev) return VTM_E_NULL;
  // y's rows are written as 16-byte vectors of eight channels
  if (C % 8 != 0 || reinterpret_cast<uintptr_t>(y_dev) % 16 != 0 || reinterpret_cast<uintptr_t>(stats_dev) % 8 != 0)
    return VTM_E_SHAPE;
  if (n > 65535 || (C + 63) / 64 > 65535) return VTM_E_SHAPE;
  const int vec_ok = HW % 8 == 0 && reinterpret_cast<uintptr_t>(x_dev) % 16 == 0;
  const dim3 grid((HW + 63) / 64, (C + 63) / 64, n);
  group_norm_tokens_kernel<<<grid, GT_THREADS, 0, static_cast<cudaStream_t>(stream_)>>>(
      static_cast<const __half*>(x_dev), stats_dev, static_cast<const __half*>(gamma_dev),
      static_cast<const __half*>(beta_dev), C, HW, groups, vec_ok, static_cast<__half*>(y_dev));
  return launch_rc();
}
