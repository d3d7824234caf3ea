// Projection GEMM of KD: D[M, N] = A[M, K] * W[N, K]^T (+ bias[N]), fp16 in / fp32 accumulate / fp16 out,
// i.e. torch.nn.Linear on fp16 tensors (to_q / to_k / to_v / to_out[0] of the attention module the
// reference calls at vidtome/patch.py:157-162).  Uses the shared wgmma mainloop; the epilogue converts
// each thread's accumulator row to fp16 and stores it through gemm::warp_store_rows64.
#include "gemm_sm90.cuh"

namespace vtm {
namespace {

struct StoreEpi {
  static constexpr uint32_t SCRATCH_PER_WARP = gemm::STAGE_STORE_BYTES;
  static constexpr bool WHOLE_ROWS = false;
  __half* d;
  const __half* bias;
  const __half* resid;   // optional [M, N] (row stride ldr): D = fp16(fp16(acc + bias) + resid), torch's `lin(x) + h`
  long long ldd, ldr;
  int M, N;
  int row0;            // first of the warp's 32 rows
  uint32_t scratch;

  __device__ __forceinline__ void set_scratch(uint32_t a) { scratch = a; }
  __device__ __forceinline__ void begin(int m_tile, int, int row_in_tile) {
    row0 = m_tile * gemm::BM + (row_in_tile & ~31);
  }
  // As in HeadSplitEpi (attention.cu): whatever is the same for the warp's 32 rows or the chunk's 64 columns is tested
  // once (warp-uniformly) and the common case — a full chunk inside N, all rows inside M — runs without per-store range
  // checks.
  __device__ __forceinline__ void tile(const gemm::Acc& acc, int col0, int ncols) {
    const int sub = threadIdx.x & 7;
#pragma unroll 1
    for (int cb = 0; cb < ncols; cb += 64) {
      uint32_t r[64];
      acc.ld64(cb, r);
      uint32_t pk[32];
      const int c0 = col0 + cb;
      const bool full = c0 + 64 <= N && ncols - cb >= 64;       // every column of the chunk exists
      if (bias) {
#pragma unroll
        for (int v8 = 0; v8 < 8; ++v8) {         // eight columns at a time: one 16-byte bias load (N % 8 == 0)
          uint4 bv = make_uint4(0, 0, 0, 0);
          if (full || c0 + 8 * v8 < N) bv = __ldg(reinterpret_cast<const uint4*>(bias + c0 + 8 * v8));
          const __half2* b2 = reinterpret_cast<const __half2*>(&bv);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float2 bf = __half22float2(b2[e]);
            pk[4 * v8 + e] = pack_f16x2(__fadd_rn(__uint_as_float(r[8 * v8 + 2 * e]), bf.x),
                                        __fadd_rn(__uint_as_float(r[8 * v8 + 2 * e + 1]), bf.y));
          }
        }
      } else {
#pragma unroll
        for (int e = 0; e < 32; ++e) pk[e] = pack_f16x2(__uint_as_float(r[2 * e]), __uint_as_float(r[2 * e + 1]));
      }
      // store phase: this lane writes columns [c, c + 8) of rows row0 + lane / 8 + 4 i
      const int c = c0 + sub * 8;
      const bool c_ok = full || (c < N && sub * 8 < ncols - cb);
      int row = row0 + ((threadIdx.x & 31) >> 3);
      __half* dst = d + static_cast<long long>(row) * ldd + c;
      const __half* rs = resid ? resid + static_cast<long long>(row) * ldr + c : nullptr;
      const long long row_step = 4 * ldd, rrow_step = 4 * ldr;
      if (row0 + 31 < M && full) {               // warp-uniform: every row and column of the chunk exists (the staging
                                                 // inside warp_store_rows64 needs the whole warp on the same path)
        if (rs) {
          gemm::warp_store_rows64(scratch, pk, [&](int, int, const uint4& v) {
            uint4 o = v;
            const uint4 rv = *reinterpret_cast<const uint4*>(rs);
            __half2* a = reinterpret_cast<__half2*>(&o);
            const __half2* b2 = reinterpret_cast<const __half2*>(&rv);
#pragma unroll
            for (int e = 0; e < 4; ++e) a[e] = __hadd2(a[e], b2[e]);
            *reinterpret_cast<uint4*>(dst) = o;
            dst += row_step;
            rs += rrow_step;
          });
        } else {
          gemm::warp_store_rows64(scratch, pk, [&](int, int, const uint4& v) {
            *reinterpret_cast<uint4*>(dst) = v;
            dst += row_step;
          });
        }
      } else {
        gemm::warp_store_rows64(scratch, pk, [&](int, int, const uint4& v) {
          if (row < M && c_ok) {
            uint4 o = v;
            if (rs) {
              const uint4 rv = *reinterpret_cast<const uint4*>(rs);
              __half2* a = reinterpret_cast<__half2*>(&o);
              const __half2* b2 = reinterpret_cast<const __half2*>(&rv);
#pragma unroll
              for (int e = 0; e < 4; ++e) a[e] = __hadd2(a[e], b2[e]);
            }
            *reinterpret_cast<uint4*>(dst) = o;
          }
          row += 4;
          dst += row_step;
          if (rs) rs += rrow_step;
        });
      }
    }
  }
  __device__ __forceinline__ void end(int, int, int) {}
};

// StoreEpi's arithmetic with the output (and the optional residual) in NCHW: GEMM row m = i HW + p is token p of sample
// i, and D[i, o, p] = fp16(fp16(acc + bias[o]) + R[i, o, p]) for D, R [n, N, HW] contiguous.  This is the exit of
// diffusers' Transformer2DModel.forward (proj_out, the permute back to NCHW and `+ residual`).
// A thread holds one token, so for one channel a warp covers only 64 contiguous bytes of D.  The two warps that hold the
// same 64 columns of a warpgroup's 64 rows therefore share their two staging areas (8 KB) as S[channel][token], 128
// bytes per channel: each thread writes its 64 values as 2-byte stores (a warp's lanes are consecutive tokens: 64
// contiguous bytes, no bank conflict), the 64 threads meet at a named barrier, and thread t then takes the 16-byte
// chunk t % 8 (eight tokens) of channels t / 8 + 8 j, so that eight lanes write (and read R) one channel's 128 bytes.
// The chunk's place in D follows from its first token alone, (m / HW, m % HW), computed once per work item: with
// HW % 8 == 0 a chunk never straddles a sample, whatever the M tile does.  Otherwise (HW = 1, or D / R not 16-byte
// aligned) each of the eight tokens is placed and stored on its own.
struct NchwEpi {
  static constexpr uint32_t SCRATCH_PER_WARP = gemm::STAGE_STORE_BYTES;
  static constexpr bool WHOLE_ROWS = false;
  __half* d;
  const __half* bias;
  const __half* resid;   // optional, laid out as d
  int M, N, HW;
  int vec_ok;            // HW % 8 == 0 and d, resid 16-byte aligned
  int m_chunk;           // first of this thread's eight tokens in the store phase
  long long off_chunk;   // (m_chunk / HW) N HW + m_chunk % HW
  uint32_t scratch;      // the pair's 8 KB

  __device__ __forceinline__ void set_scratch(uint32_t a) { scratch = a - ((threadIdx.x >> 5) & 1) * SCRATCH_PER_WARP; }
  __device__ __forceinline__ void begin(int m_tile, int, int row_in_tile) {
    m_chunk = m_tile * gemm::BM + (row_in_tile & ~63) + 8 * (threadIdx.x & 7);
    const int i = m_chunk / HW;
    off_chunk = static_cast<long long>(i) * N * HW + (m_chunk - i * HW);
  }
  __device__ __forceinline__ void tile(const gemm::Acc& acc, int col0, int ncols) {
    const int t64 = threadIdx.x & 63;
    // barriers 1 and 2 are the mainloop's: 3 + 2 (consumer warpgroup) + (column half)
    const uint32_t bar = 3 + 2 * ((threadIdx.x >> 7) - 1) + ((threadIdx.x >> 6) & 1);
#pragma unroll 1
    for (int cb = 0; cb < ncols; cb += 64) {
      uint32_t r[64];
      acc.ld64(cb, r);
      const int c0 = col0 + cb;
      const uint32_t col = scratch + 2u * t64;                 // S[0][this thread's token]
#pragma unroll
      for (int v8 = 0; v8 < 8; ++v8) {
        // without a bias the addend is -0, and acc + (-0) is acc bit for bit (+0 would turn a -0 accumulator into +0):
        // one code path, the same bits as StoreEpi's two
        uint4 bv = make_uint4(0x80008000u, 0x80008000u, 0x80008000u, 0x80008000u);
        if (bias && c0 + 8 * v8 < N) bv = __ldg(reinterpret_cast<const uint4*>(bias + c0 + 8 * v8));
        const __half2* b2 = reinterpret_cast<const __half2*>(&bv);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 bf = __half22float2(b2[e]);
          const int c = 8 * v8 + 2 * e;
          const uint32_t pk = pack_f16x2(__fadd_rn(__uint_as_float(r[c]), bf.x), __fadd_rn(__uint_as_float(r[c + 1]), bf.y));
          asm volatile("st.shared.u16 [%0], %1;" ::"r"(col + 128u * c), "h"(static_cast<uint16_t>(pk & 0xffffu)) : "memory");
          asm volatile("st.shared.u16 [%0], %1;" ::"r"(col + 128u * (c + 1)), "h"(static_cast<uint16_t>(pk >> 16)) : "memory");
        }
      }
      bar_sync_named(bar, 64);
      const int lim = min(N - c0, ncols - cb);                  // channels of this chunk that exist
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int ch = 8 * j + (t64 >> 3);
        if (ch >= lim || m_chunk >= M) continue;
        uint4 v;
        asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
                     : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                     : "r"(scratch + 128u * ch + 16u * (t64 & 7))
                     : "memory");
        const long long ch_off = static_cast<long long>(c0 + ch) * HW;
        if (vec_ok) {
          const long long o = off_chunk + ch_off;
          if (resid) {
            const uint4 rv = *reinterpret_cast<const uint4*>(resid + o);
            __half2* a = reinterpret_cast<__half2*>(&v);
            const __half2* b2 = reinterpret_cast<const __half2*>(&rv);
#pragma unroll
            for (int e = 0; e < 4; ++e) a[e] = __hadd2(a[e], b2[e]);
          }
          *reinterpret_cast<uint4*>(d + o) = v;
        } else {
          const __half* h = reinterpret_cast<const __half*>(&v);
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            const int m = m_chunk + e;
            if (m >= M) break;
            const int i = m / HW;
            const long long o = static_cast<long long>(i) * N * HW + (m - i * HW) + ch_off;
            d[o] = resid ? __hadd(h[e], resid[o]) : h[e];
          }
        }
      }
      bar_sync_named(bar, 64);                                  // S may be overwritten
    }
  }
  __device__ __forceinline__ void end(int, int, int) {}
};

// gelu(g) = 0.5 g (1 + erf(g / sqrt 2)) with ONE MUFU op: for t = |g|, log2(erfc(t / sqrt 2)) is smooth and close to a
// parabola, so h = erfc(t / sqrt 2) / 2 = 2^(p(t) - 1) with a degree-7 polynomial p (p(0) = 0), fitted minimax to
// log2(erfc(t / sqrt 2)) on [0, 5.94].  The fit bounds the exponent's absolute error (5.7e-6), i.e. h's RELATIVE error
// (4e-6), so g h stays accurate in the negative tail where h is tiny.  t is not clamped: past 5.94 p keeps falling
// (its leading coefficient is negative and it is monotonic up to 65504, with no fp32 overflow), so |g| h < 2^-26 and
// g h rounds to -0 in fp16 as gelu does, and ex2 flushes h to 0 once p < -126.  Holding h at its value at a clamp instead
// would let g h grow with |g|.  Then gelu(g) = g (1 - h) for g >= 0 and g h for g < 0: over every finite fp16 gate the
// fp16 result is within one ulp of the correctly rounded gelu, and zero wherever that is (+0 at g = -0).  At g = +inf
// p = -inf and h = 0, so g h = inf 0 = NaN: wherever h is 0 the positive branch returns g itself (the same bits for
// every finite g, since g - g 0 = g), which makes gelu(+inf) = +inf as torch's erf form gives; gelu(-inf) = -inf 0 and
// gelu(NaN) stay NaN, as there.  Two values at a time, their Horner steps interleaved.
__device__ __forceinline__ void gelu_x2(float g0, float g1, float& y0, float& y1) {
  const float t0 = fabsf(g0), t1 = fabsf(g1);
  const float lead = -1.79155074e-06f;
  float p0 = lead, p1 = lead;
  auto horner = [&](float c) {                    // p = p t + c
    p0 = __fmaf_rn(p0, t0, c);
    p1 = __fmaf_rn(p1, t1, c);
  };
  horner(6.06881658e-05f);
  horner(-0.000922937703f);
  horner(0.00847607013f);
  horner(-0.0538897403f);
  horner(-0.458542407f);
  horner(-1.15121424f);
  horner(-1.f);                                   // p(t) - 1
  const float h0 = ex2_approx(p0), h1 = ex2_approx(p1);                 // erfc(t / sqrt 2) / 2
  const float gh0 = g0 * h0, gh1 = g1 * h1;
  y0 = g0 >= 0.f ? (h0 == 0.f ? g0 : g0 - gh0) : gh0;
  y1 = g1 >= 0.f ? (h1 == 0.f ? g1 : g1 - gh1) : gh1;
}

struct GegluEpi {
  static constexpr uint32_t SCRATCH_PER_WARP = gemm::STAGE_STORE_BYTES;
  // a 64-wide output store needs 128 GEMM columns ([a32|g32] twice): each thread takes its whole 128-column row
  static constexpr bool WHOLE_ROWS = true;
  __half* d;             // [M, N/2]
  const __half* bias;    // [N], interleaved like the weight rows (may be null)
  long long ldd;
  int M, N;              // N = GEMM width (2 x output width), N % 64 == 0
  int row0;
  uint32_t scratch;

  __device__ __forceinline__ void set_scratch(uint32_t a) { scratch = a; }
  __device__ __forceinline__ void begin(int m_tile, int, int row_in_tile) {
    row0 = m_tile * gemm::BM + (row_in_tile & ~31);
  }
  __device__ __forceinline__ void tile(const gemm::Acc& acc, int col0, int ncols) {
    // two 64-column loads ([a32|g32] twice) give 64 outputs = one staged store of 32 rows x 64 columns
#pragma unroll 1
    for (int cb = 0; cb < ncols; cb += 128) {
      uint32_t pk[32];
#pragma unroll
      for (int hlf = 0; hlf < 2; ++hlf) {
        uint32_t r[64];
        acc.ld64(cb + 64 * hlf, r);
        const int c0 = col0 + cb + 64 * hlf;
#pragma unroll
        for (int v8 = 0; v8 < 4; ++v8) {       // eight values + their eight gates at a time: two 16-byte bias loads
          uint4 ba = make_uint4(0, 0, 0, 0), bg = ba;
          if (bias && c0 < N) {
            ba = __ldg(reinterpret_cast<const uint4*>(bias + c0 + 8 * v8));
            bg = __ldg(reinterpret_cast<const uint4*>(bias + c0 + 32 + 8 * v8));
          }
          const __half2* ba2 = reinterpret_cast<const __half2*>(&ba);
          const __half2* bg2 = reinterpret_cast<const __half2*>(&bg);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int i = 8 * v8 + 2 * e;
            const float2 fa = __half22float2(ba2[e]), fg = __half22float2(bg2[e]);
            // fp16 roundings of the unfused pipeline: projection output, gelu output, product.  The product of the two
            // fp16 values is taken by HMUL2 (the fp32 product of two fp16 numbers is exact, so one rounding to fp16
            // either way).
            const uint32_t a16 = pack_f16x2(__fadd_rn(__uint_as_float(r[i]), fa.x), __fadd_rn(__uint_as_float(r[i + 1]), fa.y));
            const uint32_t g16 = pack_f16x2(__fadd_rn(__uint_as_float(r[32 + i]), fg.x),
                                            __fadd_rn(__uint_as_float(r[32 + i + 1]), fg.y));
            const float2 gf = __half22float2(*reinterpret_cast<const __half2*>(&g16));
            float q0, q1;
            gelu_x2(gf.x, gf.y, q0, q1);
            const uint32_t q16 = pack_f16x2(q0, q1);
            const __half2 prod = __hmul2(*reinterpret_cast<const __half2*>(&a16), *reinterpret_cast<const __half2*>(&q16));
            pk[16 * hlf + 4 * v8 + e] = *reinterpret_cast<const uint32_t*>(&prod);
          }
        }
      }
      const int oc0 = (col0 + cb) >> 1;                       // first output column of this 64-wide store
      const int c = oc0 + (threadIdx.x & 7) * 8;
      int row = row0 + ((threadIdx.x & 31) >> 3);
      __half* dst = d + static_cast<long long>(row) * ldd + c;
      const long long row_step = 4 * ldd;
      const int No = N >> 1;
      if (row0 + 31 < M && oc0 + 64 <= No) {     // warp-uniform: the whole 32 x 64 block exists
        gemm::warp_store_rows64(scratch, pk, [&](int, int, const uint4& v) {
          *reinterpret_cast<uint4*>(dst) = v;
          dst += row_step;
        });
      } else {
        gemm::warp_store_rows64(scratch, pk, [&](int, int, const uint4& v) {
          if (row < M && c < No) *reinterpret_cast<uint4*>(dst) = v;
          row += 4;
          dst += row_step;
        });
      }
    }
  }
  __device__ __forceinline__ void end(int, int, int) {}
};

}  // namespace
}  // namespace vtm

namespace vtm {
namespace {
// Argument checks of the store GEMM (linear_impl) and of the GEGLU GEMM (geglu_impl), also run by the LoRA entry points
// before their first launch.
int linear_args(const void* a_dev, const void* w_dev, const void* resid_dev, long long ldr, int M, int N, int K,
                const void* d_dev, long long ldd) {
  if (!a_dev || !w_dev || !d_dev) return VTM_E_NULL;
  if (M <= 0 || N <= 0 || K <= 0 || (K % 8) != 0 || (N % 8) != 0 || (ldd % 8) != 0 || ldd < N) return VTM_E_SHAPE;
  if (resid_dev && ((ldr % 8) != 0 || ldr < N)) return VTM_E_SHAPE;
  return VTM_OK;
}

int geglu_args(const void* a_dev, const void* w_il_dev, int M, int N, int K, const void* d_dev, long long ldd) {
  if (!a_dev || !w_il_dev || !d_dev) return VTM_E_NULL;
  if (M <= 0 || N <= 0 || K <= 0 || (K % 8) != 0 || (N % 64) != 0 || (ldd % 8) != 0 || ldd < N / 2) return VTM_E_SHAPE;
  return VTM_OK;
}

// t_dev / u_dev / R: the K tail (T [M, R], U [N, R]); R == 0 runs the plain mainloop
int linear_impl(const void* a_dev, const void* w_dev, const void* bias_dev, const void* resid_dev, long long ldr,
                int M, int N, int K, void* d_dev, long long ldd, cudaStream_t stream, const void* t_dev = nullptr,
                const void* u_dev = nullptr, int R = 0) {
  int rc = linear_args(a_dev, w_dev, resid_dev, ldr, M, N, K, d_dev, ldd);
  if (rc) return rc;
  int sms = 0;
  rc = gemm::device_sms(&sms);
  if (rc) return rc;
  StoreEpi epi;
  epi.d = static_cast<__half*>(d_dev);
  epi.bias = static_cast<const __half*>(bias_dev);
  epi.resid = static_cast<const __half*>(resid_dev);
  epi.ldd = ldd; epi.ldr = ldr; epi.M = M; epi.N = N; epi.row0 = 0; epi.scratch = 0;
  CUtensorMap ta, tb;
  rc = make_tmap_3d_f16(&ta, a_dev, K, M, 1, K, static_cast<uint64_t>(M) * K, gemm::BK, gemm::BM);
  if (rc) return rc;
  rc = make_tmap_3d_f16(&tb, w_dev, K, N, 1, K, static_cast<uint64_t>(N) * K, gemm::BK, gemm::BN);
  if (rc) return rc;
  gemm::Work wk;
  wk.plan(M, N, K, 1, sms, 16, 1);
  wk.n_fastest = 1;
  if (R == 0) return gemm::launch<StoreEpi>(ta, tb, wk, epi, sms, stream);
  CUtensorMap tt, tu;
  rc = gemm::make_tail(t_dev, u_dev, R, M, N, &tt, &tu, &wk);
  if (rc) return rc;
  return gemm::launch_tail<StoreEpi>(ta, tb, tt, tu, wk, epi, sms, stream);
}

int geglu_impl(const void* a_dev, const void* w_il_dev, const void* bias_il_dev, int M, int N, int K, void* d_dev,
               long long ldd, cudaStream_t stream, const void* t_dev = nullptr, const void* u_il_dev = nullptr,
               int R = 0) {
  int rc = geglu_args(a_dev, w_il_dev, M, N, K, d_dev, ldd);
  if (rc) return rc;
  int sms = 0;
  rc = gemm::device_sms(&sms);
  if (rc) return rc;
  GegluEpi epi;
  epi.d = static_cast<__half*>(d_dev);
  epi.bias = static_cast<const __half*>(bias_il_dev);
  epi.ldd = ldd; epi.M = M; epi.N = N; epi.row0 = 0; epi.scratch = 0;
  CUtensorMap ta, tb;
  rc = make_tmap_3d_f16(&ta, a_dev, K, M, 1, K, static_cast<uint64_t>(M) * K, gemm::BK, gemm::BM);
  if (rc) return rc;
  rc = make_tmap_3d_f16(&tb, w_il_dev, K, N, 1, K, static_cast<uint64_t>(N) * K, gemm::BK, gemm::BN);
  if (rc) return rc;
  gemm::Work wk;
  wk.plan(M, N, K, 1, sms, 16, 1);
  wk.n_fastest = 1;
  if (R == 0) return gemm::launch<GegluEpi>(ta, tb, wk, epi, sms, stream);
  CUtensorMap tt, tu;
  rc = gemm::make_tail(t_dev, u_il_dev, R, M, N, &tt, &tu, &wk);
  if (rc) return rc;
  return gemm::launch_tail<GegluEpi>(ta, tb, tt, tu, wk, epi, sms, stream);
}

int linear_nchw_impl(const void* a_dev, const void* w_dev, const void* bias_dev, const void* resid_dev, int n, int HW,
                     int N, int K, void* d_dev, cudaStream_t stream) {
  if (!a_dev || !w_dev || !d_dev) return VTM_E_NULL;
  if (n <= 0 || HW <= 0 || N <= 0 || K <= 0 || (K % 8) != 0 || (N % 8) != 0) return VTM_E_SHAPE;
  const long long M = static_cast<long long>(n) * HW;
  if (M > 0x7fffffffLL - gemm::BM) return VTM_E_SHAPE;
  if (reinterpret_cast<uintptr_t>(d_dev) % 2 != 0 || reinterpret_cast<uintptr_t>(resid_dev) % 2 != 0) return VTM_E_SHAPE;
  int sms = 0;
  int rc = gemm::device_sms(&sms);
  if (rc) return rc;
  NchwEpi epi;
  epi.d = static_cast<__half*>(d_dev);
  epi.bias = static_cast<const __half*>(bias_dev);
  epi.resid = static_cast<const __half*>(resid_dev);
  epi.M = static_cast<int>(M); epi.N = N; epi.HW = HW;
  epi.vec_ok = HW % 8 == 0 && reinterpret_cast<uintptr_t>(d_dev) % 16 == 0 &&
               reinterpret_cast<uintptr_t>(resid_dev) % 16 == 0;
  epi.m_chunk = 0; epi.off_chunk = 0; epi.scratch = 0;
  CUtensorMap ta, tb;
  rc = make_tmap_3d_f16(&ta, a_dev, K, M, 1, K, static_cast<uint64_t>(M) * K, gemm::BK, gemm::BM);
  if (rc) return rc;
  rc = make_tmap_3d_f16(&tb, w_dev, K, N, 1, K, static_cast<uint64_t>(N) * K, gemm::BK, gemm::BN);
  if (rc) return rc;
  gemm::Work wk;
  wk.plan(static_cast<int>(M), N, K, 1, sms, 16, 1);
  wk.n_fastest = 1;
  return gemm::launch<NchwEpi>(ta, tb, wk, epi, sms, stream);
}

// Checks a LoRA descriptor and its workspace for a GEMM with M rows; *R_out = its rank (0 for no LoRA).
int lora_args(const vtm_lora_t* lora, int M, const void* ws_dev, size_t ws_bytes, int* R_out) {
  *R_out = 0;
  if (!lora || lora->R == 0) return VTM_OK;
  if (!lora->down_dev || !lora->up_dev || !ws_dev) return VTM_E_NULL;
  if (lora->R < 0 || lora->R % 8 != 0) return VTM_E_SHAPE;
  if (ws_bytes < vtm_linear_lora_workspace_bytes(M, lora->R)) return VTM_E_WS;
  // T and U are read through tensor maps: 16-byte aligned (D is checked when its map is made, before any launch)
  if (reinterpret_cast<uintptr_t>(ws_dev) % 16 != 0 || reinterpret_cast<uintptr_t>(lora->up_dev) % 16 != 0)
    return VTM_E_SHAPE;
  *R_out = lora->R;
  return VTM_OK;
}

// T = fp16(a D^T) [M, R] into the workspace, for the K tail of a LoRA-adapted projection (arguments checked).
int lora_down(const vtm_lora_t* lora, const void* a_dev, int M, int K, void* ws_dev, cudaStream_t stream) {
  return linear_impl(a_dev, lora->down_dev, nullptr, nullptr, 0, M, lora->R, K, ws_dev, lora->R, stream);
}
}  // namespace
}  // namespace vtm

extern "C" int vtm_linear_f16(const void* a_dev, const void* w_dev, const void* bias_dev, int32_t M, int32_t N,
                              int32_t K, void* d_dev, int64_t ldd, void* stream_) {
  return vtm::linear_impl(a_dev, w_dev, bias_dev, nullptr, 0, M, N, K, d_dev, ldd, static_cast<cudaStream_t>(stream_));
}

extern "C" int vtm_linear_residual_f16(const void* a_dev, const void* w_dev, const void* bias_dev, const void* resid_dev,
                                       int64_t ldr, int32_t M, int32_t N, int32_t K, void* d_dev, int64_t ldd,
                                       void* stream_) {
  if (!resid_dev) return VTM_E_NULL;
  return vtm::linear_impl(a_dev, w_dev, bias_dev, resid_dev, ldr, M, N, K, d_dev, ldd, static_cast<cudaStream_t>(stream_));
}

extern "C" int vtm_linear_nchw_residual_f16(const void* a_dev, const void* w_dev, const void* bias_dev,
                                            const void* resid_dev, int32_t n, int32_t HW, int32_t N, int32_t K,
                                            void* d_dev, void* stream_) {
  return vtm::linear_nchw_impl(a_dev, w_dev, bias_dev, resid_dev, n, HW, N, K, d_dev, static_cast<cudaStream_t>(stream_));
}

extern "C" int vtm_linear_geglu_f16(const void* a_dev, const void* w_il_dev, const void* bias_il_dev, int32_t M,
                                    int32_t N, int32_t K, void* d_dev, int64_t ldd, void* stream_) {
  return vtm::geglu_impl(a_dev, w_il_dev, bias_il_dev, M, N, K, d_dev, ldd, static_cast<cudaStream_t>(stream_));
}

extern "C" size_t vtm_linear_lora_workspace_bytes(int32_t M, int32_t R) {
  if (M <= 0 || R <= 0) return 0;
  return static_cast<size_t>(M) * R * 2;
}

extern "C" int vtm_linear_lora_f16(const void* a_dev, const void* w_dev, const void* bias_dev, const void* resid_dev,
                                   int64_t ldr, const vtm_lora_t* lora, int32_t M, int32_t N, int32_t K, void* d_dev,
                                   int64_t ldd, void* ws_dev, size_t ws_bytes, void* stream_) {
  using namespace vtm;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int rc = linear_args(a_dev, w_dev, resid_dev, ldr, M, N, K, d_dev, ldd);
  if (rc) return rc;
  int R = 0;
  rc = lora_args(lora, M, ws_dev, ws_bytes, &R);
  if (rc) return rc;
  if (R) {
    rc = lora_down(lora, a_dev, M, K, ws_dev, stream);
    if (rc) return rc;
  }
  return linear_impl(a_dev, w_dev, bias_dev, resid_dev, ldr, M, N, K, d_dev, ldd, stream, ws_dev,
                     R ? lora->up_dev : nullptr, R);
}

extern "C" int vtm_linear_geglu_lora_f16(const void* a_dev, const void* w_il_dev, const void* bias_il_dev,
                                         const vtm_lora_t* lora, int32_t M, int32_t N, int32_t K, void* d_dev,
                                         int64_t ldd, void* ws_dev, size_t ws_bytes, void* stream_) {
  using namespace vtm;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int rc = geglu_args(a_dev, w_il_dev, M, N, K, d_dev, ldd);
  if (rc) return rc;
  int R = 0;
  rc = lora_args(lora, M, ws_dev, ws_bytes, &R);
  if (rc) return rc;
  if (R) {
    rc = lora_down(lora, a_dev, M, K, ws_dev, stream);
    if (rc) return rc;
  }
  return geglu_impl(a_dev, w_il_dev, bias_il_dev, M, N, K, d_dev, ldd, stream, ws_dev, R ? lora->up_dev : nullptr, R);
}
