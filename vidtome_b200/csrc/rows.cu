// HBM-bound row kernels: K0 normalise+split, KC merge gather, KE unmerge gather + residual add.
// All three move whole token rows (C fp16, C % 8 == 0) with 16-byte vector accesses.  A row is owned by
// a group of G lanes (G = 8/16/32 chosen so that each lane holds <= 5..8 vectors of the row in registers),
// so a warp works on 32/G rows at once with all their loads in flight, the row-index lookup is done once
// per row, and reductions over a row are G-lane shuffles.  Grids are a multiple of the SM count and
// stride over rows.
//
// K0 and KC can apply the block's LayerNorm (norm1, vidtome/patch.py:146) on the fly to the rows they read:
// the row is already in registers, so norm1's output never has to be written to and re-read from HBM.
// The fused LayerNorm follows torch's half kernel: statistics in fp32, y = gamma * (rstd * (x - mean)) + beta
// in fp32, rounded to fp16 — and only then used (K0 goes on to L2-normalise the rounded row, as
// merge.py:84 does with norm1's fp16 output).
#include "common.cuh"
#include "ptx.cuh"

namespace vtm {
namespace {

constexpr int ROW_THREADS = 256;

__device__ __forceinline__ uint4 ld_nc_16(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ void st_16(void* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(v.x), "r"(v.y),
               "r"(v.z), "r"(v.w)
               : "memory");
}

template <int G>
__device__ __forceinline__ float group_sum(float v) {
#pragma unroll
  for (int o = G / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

struct LnParams {
  const __half* w;   // gamma [C] (nullptr = no LayerNorm)
  const __half* b;   // beta  [C] (may be nullptr)
  float eps;
};

// In-register LayerNorm of one row held as P vectors per lane by a G-lane group (torch half semantics: fp32
// statistics, y = gamma * (rstd * (x - mean)) + beta in fp32, rounded to fp16).  To keep the instruction count of the
// kernels that fuse it down, the row is converted to fp32 ONCE and kept in registers through both statistics
// passes and the affine step, and gamma / beta are read as fp32 from shared memory (staged once per CTA by
// stage_ln_params) instead of two 16-byte global loads + 16 conversions per data vector.
constexpr int LN_MAX_C = 2048;
__device__ __forceinline__ void stage_ln_params(const LnParams& ln, int C, float* s_gamma, float* s_beta) {
  for (int i = threadIdx.x; i < C; i += blockDim.x) {
    s_gamma[i] = __half2float(ln.w[i]);
    s_beta[i] = ln.b ? __half2float(ln.b[i]) : 0.f;
  }
  __syncthreads();
}
// Sum of two pairs of partial sums (x, y): the lanes first, then the two lane totals.
__device__ __forceinline__ float pair_sum(float2 a, float2 b) { return __fadd_rn(a.x, b.x) + __fadd_rn(a.y, b.y); }
// The row lives in registers as P x 4 fp32 pairs, one per fp16 pair of a vector.
// FULL: the row is exactly G x P vectors wide (C = 320 / 640 / 1280 with G = 8 / 16 / 32, P = 5), so the per-vector range
// tests — a divergence scaffold of BSSY / BSYNC / BRA around every vector in SASS — are compiled out.
template <int G, int P, bool FULL = false>
__device__ __forceinline__ void layer_norm_row(uint4 (&v)[P], int sub, int vecs, int C, float eps,
                                               const float* __restrict__ s_gamma, const float* __restrict__ s_beta) {
  float2 f[P][4];
  float2 acc[2] = {{0.f, 0.f}, {0.f, 0.f}};
#pragma unroll
  for (int i = 0; i < P; ++i) {
    const __half2* h = reinterpret_cast<const __half2*>(&v[i]);   // vectors beyond the row were loaded as zeros
#pragma unroll
    for (int e = 0; e < 4; ++e) f[i][e] = __half22float2(h[e]);
#pragma unroll
    for (int e = 0; e < 4; e += 2) {
      acc[e / 2].x = __fadd_rn(acc[e / 2].x, __fadd_rn(f[i][e].x, f[i][e + 1].x));
      acc[e / 2].y = __fadd_rn(acc[e / 2].y, __fadd_rn(f[i][e].y, f[i][e + 1].y));
    }
  }
  const float mean = group_sum<G>(pair_sum(acc[0], acc[1])) / static_cast<float>(C);
  float2 q[2] = {{0.f, 0.f}, {0.f, 0.f}};
#pragma unroll
  for (int i = 0; i < P; ++i) {
    if (FULL || sub + G * i < vecs) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        f[i][e].x = __fadd_rn(f[i][e].x, -mean);
        f[i][e].y = __fadd_rn(f[i][e].y, -mean);
      }
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        q[e & 1].x = __fmaf_rn(f[i][e].x, f[i][e].x, q[e & 1].x);
        q[e & 1].y = __fmaf_rn(f[i][e].y, f[i][e].y, q[e & 1].y);
      }
    }
  }
  const float rstd = rsqrtf(group_sum<G>(pair_sum(q[0], q[1])) / static_cast<float>(C) + eps);
  auto affine = [&](float x, float g, float b) { return __fmaf_rn(g, __fmul_rn(rstd, x), b); };
#pragma unroll
  for (int i = 0; i < P; ++i) {
    const int vi = sub + G * i;
    if (FULL || vi < vecs) {
      const float4 g0 = *reinterpret_cast<const float4*>(s_gamma + vi * 8), g1 = *reinterpret_cast<const float4*>(s_gamma + vi * 8 + 4);
      const float4 b0 = *reinterpret_cast<const float4*>(s_beta + vi * 8), b1 = *reinterpret_cast<const float4*>(s_beta + vi * 8 + 4);
      __half2* h = reinterpret_cast<__half2*>(&v[i]);
      h[0] = __floats2half2_rn(affine(f[i][0].x, g0.x, b0.x), affine(f[i][0].y, g0.y, b0.y));
      h[1] = __floats2half2_rn(affine(f[i][1].x, g0.z, b0.z), affine(f[i][1].y, g0.w, b0.w));
      h[2] = __floats2half2_rn(affine(f[i][2].x, g1.x, b1.x), affine(f[i][2].y, g1.y, b1.y));
      h[3] = __floats2half2_rn(affine(f[i][3].x, g1.z, b1.z), affine(f[i][3].y, g1.w, b1.w));
    }
  }
}

// ------------------------------------------------------------------ K0: [LayerNorm] + L2-normalise + split
// merge.py:84 `metric = metric / metric.norm(dim=-1, keepdim=True)`; merge.py:76-85 split().
// torch half semantics: norm accumulates in fp32 and is rounded to fp16; the division is carried out
// in fp32 on the fp16-rounded norm and rounded to fp16.
// FULL (see layer_norm_row) removes the per-vector range tests, and the two division variants run as separate loops
// instead of a test per value pair.  Neither loop may index v at run time (see the slow one): the row must stay in
// registers, or K0 stops streaming at HBM rate.
// DC: device-count (mode 2) split, src / dst rows at the capacity's row stride (vtm_split_t mode 2)
template <int G, int P, bool LN, bool FULL = false, bool DC = false>
__global__ void __launch_bounds__(ROW_THREADS, LN ? 3 : 4)
normalize_split_kernel(const __half* __restrict__ x, long long x_bs, const int* __restrict__ rowmap,
                       long long map_bs, Split sp, int B, int C, LnParams ln, __half* __restrict__ a_out,
                       __half* __restrict__ b_out) {
  __shared__ __align__(16) float s_gamma[LN ? LN_MAX_C : 4];
  __shared__ __align__(16) float s_beta[LN ? LN_MAX_C : 4];
  if (LN) stage_ln_params(ln, C, s_gamma, s_beta);
  resolve_split<DC>(sp);
  constexpr int RPW = 32 / G;                       // rows per warp
  const int lane = threadIdx.x & 31;
  const int sub = lane % G, grp = lane / G;
  const long long warp_id = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long n_warps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  const int vecs = C >> 3;
  const long long rows_per_b = static_cast<long long>(sp.Ns) + sp.Nd;
  const long long total = rows_per_b * B;
  // per-sample row strides of a_out / b_out: the counts, or the capacity of a device-count split
  const long long lda = DC ? sp.cap : sp.Ns, ldb = DC ? sp.cap : sp.Nd;
  // where row group o0 comes from and goes to
  auto locate = [&](long long o0, const __half*& src, __half*& dst) -> bool {
    const long long o = o0 + grp;
    src = x;
    dst = a_out;
    if (o >= total) return false;
    const int b = static_cast<int>(o / rows_per_b);
    const int q = static_cast<int>(o - b * rows_per_b);
    int pos;
    if (q < sp.Ns) {
      pos = src_pos<DC>(sp, q);
      dst = a_out + (b * lda + q) * C;
    } else {
      pos = dst_pos<DC>(sp, q - sp.Ns);
      dst = b_out + (b * ldb + (q - sp.Ns)) * C;
    }
    const int row = rowmap ? rowmap[b * map_bs + pos] : pos;
    src = x + b * x_bs + static_cast<long long>(row) * C;
    return true;
  };
  auto load_row = [&](uint4 (&w)[P], const __half* src, bool live) {
#pragma unroll
    for (int i = 0; i < P; ++i) {
      w[i] = make_uint4(0, 0, 0, 0);
      if (live && (FULL || sub + G * i < vecs)) w[i] = ld_nc_16(src + (sub + G * i) * 8);
    }
  };
  for (long long o0 = warp_id * RPW; o0 < total; o0 += n_warps * RPW) {
    const __half* src;
    __half* dst;
    const bool live = locate(o0, src, dst);
    uint4 v[P];
    load_row(v, src, live);
    if (LN) layer_norm_row<G, P, FULL>(v, sub, vecs, C, ln.eps, s_gamma, s_beta);
    float2 ss[2] = {{0.f, 0.f}, {0.f, 0.f}};
#pragma unroll
    for (int i = 0; i < P; ++i) {
      const __half2* h = reinterpret_cast<const __half2*>(&v[i]);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 a = __half22float2(h[e]);
        ss[e & 1].x = __fmaf_rn(a.x, a.x, ss[e & 1].x);
        ss[e & 1].y = __fmaf_rn(a.y, a.y, ss[e & 1].y);
      }
    }
    const float ss_row = group_sum<G>(pair_sum(ss[0], ss[1]));
    const float nrm = __half2float(__float2half_rn(sqrtf(ss_row)));
    // x / nrm, correctly rounded, with ONE IEEE division per row: r = RN(1/nrm), q0 = RN(x r),
    // rem = x - q0 nrm (exact, FMA), q = RN(q0 + rem r) is RN(x / nrm) (Markstein) — checked exhaustively over
    // all fp16 numerators x 3000 fp16 norms in tests/test_host_cpu.py.  Only finite normal norms take it: sub-normal
    // norms, and a norm that overflowed fp16 (sqrt(ss) >= 65520, where r = 0 and rem = 0 * inf would be NaN), take the
    // plain division, which gives the reference's x / inf = +-0.  One unsigned compare tests 2^-14 <= nrm <= 65504
    // (nrm >= +0; NaN fails it too), as cheap as the single bound it replaced.
    const bool fast = __float_as_uint(nrm) - 0x38800000u <= 0x477FE000u - 0x38800000u;
    const float rinv = 1.0f / nrm;
    auto div = [&](float x) {
      const float q0 = __fmul_rn(x, rinv);
      return __fmaf_rn(__fmaf_rn(q0, -nrm, x), rinv, q0);
    };
    if (fast) {
#pragma unroll
      for (int i = 0; i < P; ++i) {
        if (live && (FULL || sub + G * i < vecs)) {
          __half2* h = reinterpret_cast<__half2*>(&v[i]);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float2 x = __half22float2(h[e]);
            h[e] = __floats2half2_rn(div(x.x), div(x.y));
          }
          st_16(dst + (sub + G * i) * 8, v[i]);
        }
      }
    } else {
      // Unrolled like the fast path.  A loop here would index v at run time, which puts v in local memory, and then
      // every row, slow or not, stores its vectors there (ptxas reports that frame as stack, not as spill).  With such
      // a loop K0 ran at 1.2-1.7 TB/s on H100; without it, 2.5-3.2 TB/s.
#pragma unroll
      for (int i = 0; i < P; ++i) {
        if (live && (FULL || sub + G * i < vecs)) {
          __half2* h = reinterpret_cast<__half2*>(&v[i]);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float2 f = __half22float2(h[e]);
            h[e] = __halves2half2(__float2half_rn(f.x / nrm), __float2half_rn(f.y / nrm));
          }
          st_16(dst + (sub + G * i) * 8, v[i]);
        }
      }
    }
  }
}

// ------------------------------------------------------------------ KC / KE: row gathers
// y[b, i, :] = [LN](x[b, map[b, i], :]) (+ resid[b, i, :]).
// KC can also be the producer side of the global-token exchange: `peers` lists further copies of y in OTHER GPUs'
// memory (peer-mapped over NVLink), written by the same stores — the all-gather of the merged tokens then needs no
// separate pass over them (vtm_gather_rows_peers).
constexpr int MAX_PEERS = 8;
struct PeerDsts {
  __half* p[MAX_PEERS];
  int n;
};

// DL (device length): rows i >= *len_dev of each sample are written as zeros instead of gathered.
template <int G, int P, bool ADD, bool LN, bool DL = false>
__global__ void __launch_bounds__(ROW_THREADS, LN ? 3 : 4)
gather_rows_kernel(const __half* __restrict__ x, long long x_bs, const int* __restrict__ map, long long map_bs,
                   const __half* __restrict__ resid, int B, int L, int C, LnParams ln, __half* __restrict__ y,
                   long long y_bs, PeerDsts peers, const int* __restrict__ len_dev = nullptr) {
  __shared__ __align__(16) float s_gamma[LN ? LN_MAX_C : 4];
  __shared__ __align__(16) float s_beta[LN ? LN_MAX_C : 4];
  if (LN) stage_ln_params(ln, C, s_gamma, s_beta);
  constexpr int RPW = 32 / G;
  const int lane = threadIdx.x & 31;
  const int sub = lane % G, grp = lane / G;
  const long long warp_id = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long n_warps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  const int vecs = C >> 3;
  const long long total = static_cast<long long>(B) * L;
  const int l_valid = DL ? __ldg(len_dev) : L;
  for (long long o0 = warp_id * RPW; o0 < total; o0 += n_warps * RPW) {
    const long long o = o0 + grp;
    bool live = o < total;
    const __half* src = x;
    __half* dst = y;
    int b = 0, i = 0;
    if (live) {
      b = static_cast<int>(o / L);
      i = static_cast<int>(o - static_cast<long long>(b) * L);
      dst = y + b * y_bs + static_cast<long long>(i) * C;
    }
    if (DL && live && i >= l_valid) {
#pragma unroll
      for (int k = 0; k < P; ++k)
        if (sub + G * k < vecs) st_16(dst + (sub + G * k) * 8, make_uint4(0, 0, 0, 0));
      live = false;
    }
    uint4 v[P], rr[P];
    // residual rows do not depend on the map: get them in flight before the (dependent) map lookup
    if (ADD && live) {
      const __half* rs = resid + (static_cast<long long>(b) * L + i) * C;
#pragma unroll
      for (int k = 0; k < P; ++k)
        if (sub + G * k < vecs) rr[k] = ld_nc_16(rs + (sub + G * k) * 8);
    }
    if (live) {
      const int srow = map ? map[b * map_bs + i] : i;
      src = x + b * x_bs + static_cast<long long>(srow) * C;
    }
#pragma unroll
    for (int k = 0; k < P; ++k) {
      v[k] = make_uint4(0, 0, 0, 0);
      if (live && sub + G * k < vecs) v[k] = ld_nc_16(src + (sub + G * k) * 8);
    }
    if (LN) layer_norm_row<G, P>(v, sub, vecs, C, ln.eps, s_gamma, s_beta);
#pragma unroll
    for (int i = 0; i < P; ++i) {
      if (live && sub + G * i < vecs) {
        if (ADD) {
          __half2* a = reinterpret_cast<__half2*>(&v[i]);
          const __half2* r2 = reinterpret_cast<const __half2*>(&rr[i]);
#pragma unroll
          for (int e = 0; e < 4; ++e) a[e] = __hadd2(a[e], r2[e]);
        }
        st_16(dst + (sub + G * i) * 8, v[i]);
        if (!ADD) {
          const long long off = (dst - y) + (sub + G * i) * 8;
          for (int d = 0; d < peers.n; ++d) *reinterpret_cast<uint4*>(peers.p[d] + off) = v[i];
        }
      }
    }
  }
}

int sm_count(int* sms) { return cached_sm_count(sms); }

// Grid of a grid-stride row kernel: never more CTAs than are resident at once (sms x the kernel's occupancy), so
// that all warps run the same number of iterations (+-1) instead of a short last wave.
template <class K>
int grid_for_rows(K kernel, long long rows, int rows_per_warp, int sms) {
  // occupancy per kernel (all instantiations of one template share the function-pointer TYPE, so the cache is keyed
  // by the pointer value); a handful of entries, filled once each
  static const void* known[32];
  static int occ[32];
  static int n_known = 0;
  const void* key = reinterpret_cast<const void*>(kernel);
  int per_sm = 0;
  for (int i = 0; i < n_known; ++i)
    if (known[i] == key) per_sm = occ[i];
  if (per_sm == 0) {
    int n = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kernel, ROW_THREADS, 0) != cudaSuccess || n < 1) n = 2;
    per_sm = n;
    if (n_known < 32) { known[n_known] = key; occ[n_known] = n; ++n_known; }
  }
  const long long warps = (rows + rows_per_warp - 1) / rows_per_warp;
  long long blocks = (warps + (ROW_THREADS / 32) - 1) / (ROW_THREADS / 32);
  const long long cap = static_cast<long long>(sms) * per_sm;
  if (blocks < 1) blocks = 1;
  if (blocks > cap) blocks = cap;
  return static_cast<int>(blocks);
}

// (G, P) for a row of `vecs` 16-byte vectors: G lanes x P vectors per lane >= vecs
#define VTM_DISPATCH_GP(vecs, CALL)                 \
  if ((vecs) <= 8 * 5) { CALL(8, 5) }               \
  else if ((vecs) <= 16 * 5) { CALL(16, 5) }        \
  else if ((vecs) <= 32 * 5) { CALL(32, 5) }        \
  else { CALL(32, 8) }

}  // namespace
}  // namespace vtm

extern "C" int vtm_normalize_split_ln(const void* x_dev, int64_t x_batch_stride, const int32_t* rowmap_dev,
                                      int64_t rowmap_batch_stride, const vtm_split_t* split, int32_t B,
                                      int32_t C, const void* ln_weight_dev, const void* ln_bias_dev, float ln_eps,
                                      void* a_out_dev, void* b_out_dev, void* stream_) {
  using namespace vtm;
  Split sp;
  int rc = make_split(split, &sp);
  if (rc) return rc;
  if (!x_dev || (sp.Ns > 0 && !a_out_dev) || (sp.Nd > 0 && !b_out_dev)) return VTM_E_NULL;
  if (B <= 0 || C <= 0 || (C % 8) != 0 || C > 32 * 8 * 8) return VTM_E_SHAPE;   // <= LN_MAX_C
  int sms = 0;
  rc = sm_count(&sms);
  if (rc) return rc;
  const long long rows = (static_cast<long long>(sp.Ns) + sp.Nd) * B;
  const int vecs = C / 8;
  LnParams ln{static_cast<const __half*>(ln_weight_dev), static_cast<const __half*>(ln_bias_dev), ln_eps};
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
#define CALL_K0_(G, P, LN, FULL, DC)                                                                               \
  normalize_split_kernel<G, P, LN, FULL, DC>                                                                      \
      <<<grid_for_rows(normalize_split_kernel<G, P, LN, FULL, DC>, rows, 32 / G, sms), ROW_THREADS, 0, st>>>(     \
          static_cast<const __half*>(x_dev), x_batch_stride, rowmap_dev, rowmap_batch_stride, sp, B, C, ln,       \
          static_cast<__half*>(a_out_dev), static_cast<__half*>(b_out_dev));
  if (sp.glob_len_dev) {
    // the global stage's tokens are already normalised by norm1 (KC wrote them): no fused LayerNorm on this path
    if (ln.w) return VTM_E_UNSUPPORTED;
#define CALL(G, P) CALL_K0_(G, P, false, false, true)
    VTM_DISPATCH_GP(vecs, CALL)
#undef CALL
    return launch_rc();
  }
#define CALL_K0(G, P, LN)                                   \
  if (vecs == (G) * (P)) { CALL_K0_(G, P, LN, true, false) }       \
  else { CALL_K0_(G, P, LN, false, false) }
  if (ln.w) {
#define CALL(G, P) CALL_K0(G, P, true)
    VTM_DISPATCH_GP(vecs, CALL)
#undef CALL
  } else {
#define CALL(G, P) CALL_K0(G, P, false)
    VTM_DISPATCH_GP(vecs, CALL)
#undef CALL
  }
#undef CALL_K0
#undef CALL_K0_
  return launch_rc();
}

extern "C" int vtm_normalize_split(const void* x_dev, int64_t x_batch_stride, const int32_t* rowmap_dev,
                                   int64_t rowmap_batch_stride, const vtm_split_t* split, int32_t B,
                                   int32_t C, void* a_out_dev, void* b_out_dev, void* stream_) {
  return vtm_normalize_split_ln(x_dev, x_batch_stride, rowmap_dev, rowmap_batch_stride, split, B, C, nullptr,
                                nullptr, 0.f, a_out_dev, b_out_dev, stream_);
}

extern "C" int vtm_gather_rows_peers(const void* x_dev, int64_t x_batch_stride, const int32_t* map_dev,
                                     int64_t map_batch_stride, int32_t B, int32_t L, int32_t C,
                                     const void* ln_weight_dev, const void* ln_bias_dev, float ln_eps, void* y_dev,
                                     int64_t y_batch_stride, void* const* peer_y_devs, int32_t n_peers,
                                     void* stream_) {
  using namespace vtm;
  if (!x_dev || !y_dev || (n_peers > 0 && !peer_y_devs)) return VTM_E_NULL;
  if (B <= 0 || L < 0 || C <= 0 || (C % 8) != 0 || C > 32 * 8 * 8) return VTM_E_SHAPE;
  if (n_peers < 0 || n_peers > MAX_PEERS) return VTM_E_SHAPE;
  if (L == 0) return VTM_OK;
  PeerDsts peers;
  peers.n = n_peers;
  for (int d = 0; d < MAX_PEERS; ++d) peers.p[d] = d < n_peers ? static_cast<__half*>(peer_y_devs[d]) : nullptr;
  for (int d = 0; d < n_peers; ++d)
    if (!peers.p[d]) return VTM_E_NULL;
  int sms = 0;
  int rc = sm_count(&sms);
  if (rc) return rc;
  const long long rows = static_cast<long long>(B) * L;
  const int vecs = C / 8;
  LnParams ln{static_cast<const __half*>(ln_weight_dev), static_cast<const __half*>(ln_bias_dev), ln_eps};
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
#define CALL_KC(G, P, LN)                                                                                      \
  gather_rows_kernel<G, P, false, LN>                                                                          \
      <<<grid_for_rows(gather_rows_kernel<G, P, false, LN>, rows, 32 / G, sms), ROW_THREADS, 0, st>>>(         \
          static_cast<const __half*>(x_dev), x_batch_stride, map_dev, map_batch_stride, nullptr, B, L, C, ln,  \
          static_cast<__half*>(y_dev), y_batch_stride, peers);
  if (ln.w) {
#define CALL(G, P) CALL_KC(G, P, true)
    VTM_DISPATCH_GP(vecs, CALL)
#undef CALL
  } else {
#define CALL(G, P) CALL_KC(G, P, false)
    VTM_DISPATCH_GP(vecs, CALL)
#undef CALL
  }
#undef CALL_KC
  return launch_rc();
}

extern "C" int vtm_gather_rows_ln(const void* x_dev, int64_t x_batch_stride, const int32_t* map_dev,
                                  int64_t map_batch_stride, int32_t B, int32_t L, int32_t C,
                                  const void* ln_weight_dev, const void* ln_bias_dev, float ln_eps, void* y_dev,
                                  int64_t y_batch_stride, void* stream_) {
  return vtm_gather_rows_peers(x_dev, x_batch_stride, map_dev, map_batch_stride, B, L, C, ln_weight_dev, ln_bias_dev,
                               ln_eps, y_dev, y_batch_stride, nullptr, 0, stream_);
}

extern "C" int vtm_gather_rows(const void* x_dev, int64_t x_batch_stride, const int32_t* map_dev,
                               int64_t map_batch_stride, int32_t B, int32_t L, int32_t C, void* y_dev,
                               int64_t y_batch_stride, void* stream_) {
  return vtm_gather_rows_ln(x_dev, x_batch_stride, map_dev, map_batch_stride, B, L, C, nullptr, nullptr, 0.f,
                            y_dev, y_batch_stride, stream_);
}

extern "C" int vtm_gather_rows_dev(const void* x_dev, int64_t x_batch_stride, const int32_t* map_dev,
                                   int64_t map_batch_stride, int32_t B, int32_t L_cap, int32_t C, const int32_t* len_dev,
                                   void* y_dev, int64_t y_batch_stride, void* stream_) {
  using namespace vtm;
  if (!x_dev || !y_dev || !map_dev || !len_dev) return VTM_E_NULL;
  if (B <= 0 || L_cap < 0 || C <= 0 || (C % 8) != 0 || C > 32 * 8 * 8) return VTM_E_SHAPE;
  if (L_cap == 0) return VTM_OK;
  int sms = 0;
  int rc = sm_count(&sms);
  if (rc) return rc;
  const long long rows = static_cast<long long>(B) * L_cap;
  const int vecs = C / 8;
  LnParams ln{nullptr, nullptr, 0.f};
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
#define CALL(G, P)                                                                                                \
  gather_rows_kernel<G, P, false, false, true>                                                                    \
      <<<grid_for_rows(gather_rows_kernel<G, P, false, false, true>, rows, 32 / G, sms), ROW_THREADS, 0, st>>>(   \
          static_cast<const __half*>(x_dev), x_batch_stride, map_dev, map_batch_stride, nullptr, B, L_cap, C, ln, \
          static_cast<__half*>(y_dev), y_batch_stride, PeerDsts{}, len_dev);
  VTM_DISPATCH_GP(vecs, CALL)
#undef CALL
  return launch_rc();
}

extern "C" int vtm_unmerge_add(const void* y_dev, int64_t y_batch_stride, const int32_t* map_dev,
                               int64_t map_batch_stride, const void* resid_dev, int32_t B, int32_t N,
                               int32_t C, void* out_dev, void* stream_) {
  using namespace vtm;
  if (!y_dev || !out_dev || !map_dev) return VTM_E_NULL;
  if (B <= 0 || N < 0 || C <= 0 || (C % 8) != 0 || C > 32 * 8 * 8) return VTM_E_SHAPE;
  if (N == 0) return VTM_OK;
  int sms = 0;
  int rc = sm_count(&sms);
  if (rc) return rc;
  const long long rows = static_cast<long long>(B) * N;
  const int vecs = C / 8;
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  const long long out_bs = static_cast<long long>(N) * C;
  LnParams ln{nullptr, nullptr, 0.f};
  if (resid_dev) {
#define CALL(G, P)                                                                                          \
  gather_rows_kernel<G, P, true, false>                                                                     \
      <<<grid_for_rows(gather_rows_kernel<G, P, true, false>, rows, 32 / G, sms), ROW_THREADS, 0, st>>>(    \
          static_cast<const __half*>(y_dev), y_batch_stride, map_dev, map_batch_stride,                     \
          static_cast<const __half*>(resid_dev), B, N, C, ln, static_cast<__half*>(out_dev), out_bs, PeerDsts{});
    VTM_DISPATCH_GP(vecs, CALL)
#undef CALL
  } else {
#define CALL(G, P)                                                                                          \
  gather_rows_kernel<G, P, false, false>                                                                    \
      <<<grid_for_rows(gather_rows_kernel<G, P, false, false>, rows, 32 / G, sms), ROW_THREADS, 0, st>>>(   \
          static_cast<const __half*>(y_dev), y_batch_stride, map_dev, map_batch_stride, nullptr, B, N, C, ln, \
          static_cast<__half*>(out_dev), out_bs, PeerDsts{});
    VTM_DISPATCH_GP(vecs, CALL)
#undef CALL
  }
  return launch_rc();
}
