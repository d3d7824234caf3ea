// KD — merged-token self-attention for sm_90a: QKV projection (wgmma GEMM, gemm_sm90.cuh) -> flash
// attention (this file) -> output projection (wgmma GEMM, linear.cu).
//
// Reference: `self.attn1(merged_tokens)` at vidtome/patch.py:157-162 = diffusers Attention; the math is
// restated in the reference at utils/pnp_utils.py:47-95: softmax(q k^T * scale) v per head.
//
// Flash-attention kernel (flash_attn_kernel below): one CTA per (64 x CW-row query tile, head, sample), a TMA producer
// warpgroup streaming K/V tiles of one head (contiguous runs of the head-major padded buffers written by the projection
// epilogue) through an mbarrier ring, and CW = 3 (head_dim <= 80) or 2 wgmma consumer warpgroups running S = Q K^T, the
// online softmax and O += P V with P kept in registers, each overlapping its softmax with its own P V.  A shared (PnP)
// call serves G samples per CTA with one softmax (see flash_attn_kernel); its samples are `inputs` runs of `period` frames,
// and sample f + j period reads the queries and keys of sample f.
#include <stdlib.h>

#include "gemm_sm90.cuh"

extern "C" int vtm_linear_f16(const void*, const void*, const void*, int32_t, int32_t, int32_t, void*, int64_t,
                              void*);
extern "C" int vtm_linear_residual_f16(const void*, const void*, const void*, const void*, int64_t, int32_t, int32_t,
                                       int32_t, void*, int64_t, void*);
extern "C" int vtm_linear_lora_f16(const void*, const void*, const void*, const void*, int64_t, const vtm_lora_t*,
                                   int32_t, int32_t, int32_t, void*, int64_t, void*, size_t, void*);

namespace vtm {
namespace {

// ---------------------------------------------------------------------------------------------------------
// QKV projection epilogue: writes q, k, v HEAD-MAJOR with rows padded to DP = 64, 128 or 192 halfs (fa_padded_row):
//   qkvh[which][b][head][l][0..DP)   (which = 0 q, 1 k, 2 v; columns >= head_dim are written as zeros)
// so that a K or V tile of consecutive keys of one head is one contiguous run of full cache lines (read in place
// from the [B*L, 3C] GEMM output, every key row would be an 80-byte slice at a 1920-byte pitch: many partial-sector
// L2 requests per tile).
struct HeadSplitEpi {
  static constexpr uint32_t SCRATCH_PER_WARP = gemm::STAGE_STORE_BYTES;
  static constexpr bool WHOLE_ROWS = false;
  __half* qkvh;
  int M, C, H, d, L, DP, nb; // M = nb*L rows, C = H*d
  int dread;                 // columns of a padded row that the flash kernel reads: 16 x (its k-step count) <= DP
  int which0, n_proj;        // this GEMM produces projections which0 .. which0 + n_proj - 1 of (q, k, v); N = n_proj * C
  long long which_stride;    // distance between the projections: B*H*L*DP
  int row0;                  // first of the warp's 32 rows
  int b0, l0;                // (sample, position) of row0 + lane / 8, this lane's first row in the store phase
  uint32_t scratch;

  __device__ __forceinline__ void set_scratch(uint32_t a) { scratch = a; }
  // With K = 320 / 640 this epilogue, not the MMAs, bounds the projection GEMMs: everything that is the same for the
  // warp's 32 rows or the chunk's 64 columns is decided once, warp-uniformly, and the common case (rows of one sample,
  // all in range; chunk inside one projection) runs without per-store tests.
  int bw, lw;                // (sample, position) of row0, the first of the warp's 32 rows (warp-uniform)
  float inv_c, inv_d;        // 1 / C, 1 / d (set by the host) for the exact small-integer divisions below
  __device__ __forceinline__ void begin(int m_tile, int, int row_in_tile) {
    row0 = m_tile * gemm::BM + (row_in_tile & ~31);
    bw = row0 / L;
    lw = row0 - bw * L;
    // this lane's first row in the store phase: row0 + lane / 8, up to 3 rows past row0, i.e. up to 3 samples
    // further on when L < 3 (one subtraction would leave l0 >= L at L = 1)
    b0 = bw;
    l0 = lw + ((row_in_tile & 31) >> 3);
    while (l0 >= L) { l0 -= L; ++b0; }
  }
  // exact x / y for 0 <= x < 2^22 (x + 0.5 keeps the product away from the integer boundary)
  static __device__ __forceinline__ int div_small(int x, float inv_y) {
    return static_cast<int>((static_cast<float>(x) + 0.5f) * inv_y);
  }
  __device__ __forceinline__ void tile(const gemm::Acc& acc, int col0, int ncols) {
    const int sub = threadIdx.x & 7;
    const bool rows_plain = lw + 31 < L && bw < nb;      // the warp's 32 rows exist and lie in one sample
#pragma unroll 1
    for (int cb = 0; cb < ncols; cb += 64) {
      uint32_t r[64];
      acc.ld64(cb, r);
      uint32_t pk[32];
      const int cfirst = col0 + cb;
#pragma unroll
      for (int e = 0; e < 32; ++e) pk[e] = pack_f16x2(__uint_as_float(r[2 * e]), __uint_as_float(r[2 * e + 1]));
      // this lane's 8 columns in the store phase: the same for all of its rows
      const int n = cfirst + sub * 8;                        // groups of 8 columns never straddle a head (d % 8 == 0)
      const bool n_ok = n < n_proj * C && sub * 8 < ncols - cb;
      const int which = div_small(n, inv_c), c = n - which * C;
      const int head = div_small(c, inv_d), e0 = c - head * d;
      // columns [d, dread) are read by the flash kernel's last k-step (dread = 16 x its k-step count): zeros.  The
      // padding beyond dread (up to DP) is never read, so it is NOT written.
      const bool pads = e0 + 8 == d && d < dread;
      // dst(b, l) = base + (b H L + l) DP: stepped by 4 rows per store (plus (H - 1) L DP when crossing a sample)
      __half* dst = qkvh + which * which_stride + static_cast<long long>(head) * L * DP + e0 +
                    (static_cast<long long>(b0) * H * L + l0) * DP;
      const long long row_step = 4ll * DP;
      // staged through shared memory (gemm::warp_store_rows64): eight lanes write 64 consecutive columns of one row
      if (rows_plain) {
        if (!n_ok) dst = nullptr;
        gemm::warp_store_rows64(scratch, pk, [&](int, int, const uint4& v) {
          if (dst) {
            *reinterpret_cast<uint4*>(dst) = v;
            if (pads) {
              for (int pe = d; pe < dread; pe += 8) *reinterpret_cast<uint4*>(dst + 8 + (pe - d)) = make_uint4(0, 0, 0, 0);
            }
            dst += row_step;
          }
        });
      } else {
        const long long sample_step = static_cast<long long>(H - 1) * L * DP;
        int bb = b0, ll = l0;
        gemm::warp_store_rows64(scratch, pk, [&](int, int, const uint4& v) {
          if (bb < nb && n_ok) {
            *reinterpret_cast<uint4*>(dst) = v;
            if (pads) {
              for (int pe = d; pe < dread; pe += 8) *reinterpret_cast<uint4*>(dst + 8 + (pe - d)) = make_uint4(0, 0, 0, 0);
            }
          }
          ll += 4;                                              // next row of this lane: 4 further down
          dst += row_step;
          while (ll >= L) { ll -= L; ++bb; dst += sample_step; }
        });
      }
    }
  }
  __device__ __forceinline__ void end(int, int, int) {}
};

// Columns of a head-major padded row that the flash kernel reads for head_dim d: 16 x its k-step count.
inline int fa_columns_read(int d) { return 16 * ((d + 15) / 16); }

// Largest head_dim the flash kernel is built for (KS = 10 k-steps).
constexpr int FA_MAX_HEAD_DIM = 160;

// Padded row of the head-major q / k / v buffers: the 64-column TMA boxes the flash kernel loads (64, 128 or 192 halfs).
inline int fa_padded_row(int d) { return 64 * ((fa_columns_read(d) + 63) / 64); }

// x [nb * L, K] -> projections which0 .. which0 + n_proj - 1 of (q, k, v), head-major padded, at `out`
// ([n_proj][nb][H][L][DP], or projections `which_stride` halfs apart when it is > 0); w [n_proj * C, K].
// t / u / R: a LoRA's K tail, T [nb * L, R] and U [n_proj * C, R] (R == 0: none).
int launch_head_proj(const void* x, const void* w, __half* out, int nb, int L, int K, int C, int H, int DP, int which0,
                     int n_proj, cudaStream_t stream, long long which_stride = 0, const void* t = nullptr,
                     const void* u = nullptr, int R = 0) {
  int sms = 0;
  int rc = gemm::device_sms(&sms);
  if (rc) return rc;
  const int M = nb * L, N = n_proj * C;
  HeadSplitEpi epi;
  epi.qkvh = out; epi.M = M; epi.C = C; epi.H = H; epi.d = C / H; epi.L = L; epi.DP = DP;
  epi.dread = fa_columns_read(C / H);
  epi.which0 = which0; epi.n_proj = n_proj;
  epi.which_stride = which_stride > 0 ? which_stride : static_cast<long long>(nb) * H * L * DP; epi.row0 = 0; epi.scratch = 0; epi.b0 = 0; epi.l0 = 0; epi.nb = nb;
  epi.bw = 0; epi.lw = 0; epi.inv_c = 1.f / static_cast<float>(C); epi.inv_d = 1.f / static_cast<float>(C / H);
  CUtensorMap ta, tb;
  rc = make_tmap_3d_f16(&ta, x, K, M, 1, K, static_cast<uint64_t>(M) * K, gemm::BK, gemm::BM);
  if (rc) return rc;
  rc = make_tmap_3d_f16(&tb, w, K, N, 1, K, static_cast<uint64_t>(N) * K, gemm::BK, gemm::BN);
  if (rc) return rc;
  gemm::Work wk;
  wk.plan(M, N, K, 1, sms, 16, 1);
  wk.n_fastest = 1;
  if (R == 0) return gemm::launch<HeadSplitEpi>(ta, tb, wk, epi, sms, stream);
  CUtensorMap tt, tu;
  rc = gemm::make_tail(t, u, R, M, N, &tt, &tu, &wk);
  if (rc) return rc;
  return gemm::launch_tail<HeadSplitEpi>(ta, tb, tt, tu, wk, epi, sms, stream);
}

// Rank of a LoRA descriptor (0 for NULL), checked.
int lora_rank(const vtm_lora_t* l, int* R) {
  *R = 0;
  if (!l || l->R == 0) return VTM_OK;
  if (l->R < 0 || l->R % 8 != 0) return VTM_E_SHAPE;
  if (!l->down_dev || !l->up_dev) return VTM_E_NULL;
  *R = l->R;
  return VTM_OK;
}

constexpr int FA_BKV = 64;       // keys per K/V tile

struct FaParams {
  __half* o;          // [B*Lq, C]
  int L, Lq, H, d, C, B;
  const int* len_dev; // DL: the sequence length on the device (self-attention, <= L == Lq, the buffers' row count)
  float scale_log2;   // softmax scale * log2(e)
  // Whose q and k each sample reads.  The B samples are `inputs` runs of `period` frames: sample b = f + j period (frame
  // f, input j) reads the q / k slab of sample f and its own v, and `groups` CTAs serve each frame, up to G inputs each.
  // PnP injection (utils/pnp_utils.py:57-68,87-91) on merged tokens is period 1 (every sample reads sample 0), on the
  // frames of an unmerged block period n (sample b reads sample b mod n); without sharing period = B, inputs = 1.
  int period, inputs, groups;
};

constexpr size_t FA_SMEM_MAX = 227 * 1024;   // dynamic shared memory a CTA may opt in to on sm_90

template <int KS, int G = 1>
struct FaCfg {
  // Consumer warpgroups, 64 query rows each.  Three (512 threads, at most 128 registers each) hide more of the softmax's
  // latency than two; from head_dim 96 on, O no longer fits next to S and P in 128 registers, so those keep two.  A
  // CTA that serves G > 1 samples holds G accumulators O and keeps two (up to 168 registers each, or 232 with the
  // producer's registers from head_dim 136 on: fa_moves_registers).
  static constexpr int CW = G == 1 && KS <= 5 ? 3 : 2;
  static constexpr int BQ = 64 * CW;                      // query rows per CTA
  static constexpr int THREADS = 128 * (CW + 1);          // producer warpgroup + consumers
  static constexpr int DV = 16 * KS;                      // head_dim rounded up to 16: k-steps of Q K^T, width of O
  static constexpr int ATOMS = (KS + 3) / 4;              // 64-column blocks of a padded row (one TMA box each)
  static constexpr uint32_t Q_ATOM = BQ * 128;            // [BQ rows x 128 B]
  static constexpr uint32_t KV_ATOM = FA_BKV * 128;       // [64 rows x 128 B]
  static constexpr uint32_t Q_BYTES = ATOMS * Q_ATOM;
  static constexpr uint32_t TILE_BYTES = ATOMS * KV_ATOM;
  static constexpr uint32_t STAGE_BYTES = (1 + G) * TILE_BYTES; // K + the V tiles of G samples
  // K/V ring depth.  The consumers hold two stages at a time (Q K^T of tile j+1 is issued before P V of tile j), so
  // four stages keep two tile loads in flight; five timed the same at both bench shapes.  Wide grouped stages get as
  // many as fit (three at head_dim > 64 and G = 3: one load in flight).
  static constexpr int STAGES_FIT = static_cast<int>((FA_SMEM_MAX - 1024 - Q_BYTES - 256) / STAGE_BYTES);
  static constexpr int STAGES = STAGES_FIT < 4 ? STAGES_FIT : 4;
  static_assert(STAGES >= 3, "the consumers hold two stages: a third keeps a load in flight");
  static constexpr size_t SMEM_BYTES = 1024 + Q_BYTES + static_cast<size_t>(STAGES) * STAGE_BYTES + 256;
};

// Largest number of samples one CTA serves in a shared (PnP) call at KS k-steps: G accumulators O of DV / 2 registers
// each next to S and P without spills (ptxas -v; DESIGN §4).
constexpr int fa_group_max(int KS) { return KS <= 2 ? 4 : KS == 3 ? 3 : KS <= 5 ? 2 : 1; }

// From head_dim 136 on (KS >= 9) O takes 72 or 80 registers next to S and P, which leaves KS = 10 at 167 of the 168
// that 384 threads get at launch: the producer warpgroup, one lane of which only issues TMA loads, gives its registers
// to the two consumer warpgroups (128 x 40 + 256 x 232 <= 64K), as the GEMM mainloop does.  Below that the kernels are
// built without setmaxnreg (DESIGN §4).
constexpr bool fa_moves_registers(int KS) { return KS >= 9; }

// Online softmax of one 64-key tile of S in the log2 domain.  The thread holds rows r0 = lane/4 (s[4n], s[4n+1]) and
// r0 + 8 (s[4n+2], s[4n+3]), columns 8n + 2(lane%4).  On return s holds P = ex2(s * scale - m_new), m_r the new row
// maxima, l_r the rescaled row sums with this tile's P added, alpha the factor O must be rescaled by before P V of this
// tile is added to it.  MASK (the last tile only) sets keys at or past `kvalid` to -inf.  The roundings are spelled
// out: scale as a separate multiply, then ex2 of a subtraction, and l = fma(l, alpha, p0 + p1) for the first pair.
// A row whose scores so far are all -inf (every key of its first tiles -inf, e.g. a K channel that overflowed to +inf
// against a negative query component) keeps m_r = -inf: it subtracts 0 instead, as FlashAttention-2 does, so those
// keys get p = 0 and alpha = 0 rather than ex2(-inf - -inf) = NaN.  Finite rows subtract their maximum unchanged.
// A row whose every key scores -inf ends with l = 0 and O = 0 (see the store).
template <bool MASK>
__device__ __forceinline__ void fa_softmax(float (&s)[32], float (&m_r)[2], float (&l_r)[2], float (&alpha)[2],
                                           float scale_log2, int kvalid, int lane) {
  float mx[2] = {-INFINITY, -INFINITY}, m_safe[2];
#pragma unroll
  for (int n = 0; n < 8; ++n) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      float v = __fmul_rn(s[4 * n + e], scale_log2);
      if (MASK) {
        const int col = n * 8 + 2 * (lane & 3) + (e & 1);
        v = col < kvalid ? v : -INFINITY;
      }
      s[4 * n + e] = v;
      mx[e >> 1] = fmaxf(mx[e >> 1], v);
    }
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
    const float m_new = fmaxf(m_r[r], mx[r]);   // -inf while every score of the row so far is -inf
    const float m_sub = m_new == -INFINITY ? 0.f : m_new;
    alpha[r] = ex2_approx(__fsub_rn(m_r[r], m_sub));
    m_r[r] = m_new;
    m_safe[r] = m_sub;
  }
#pragma unroll
  for (int n = 0; n < 8; ++n) {
    const float p0 = ex2_approx(__fsub_rn(s[4 * n], m_safe[0])), p1 = ex2_approx(__fsub_rn(s[4 * n + 1], m_safe[0]));
    const float p2 = ex2_approx(__fsub_rn(s[4 * n + 2], m_safe[1])), p3 = ex2_approx(__fsub_rn(s[4 * n + 3], m_safe[1]));
    if (n == 0) {
      l_r[0] = __fmaf_rn(l_r[0], alpha[0], __fadd_rn(p0, p1));
      l_r[1] = __fmaf_rn(l_r[1], alpha[1], __fadd_rn(p2, p3));
    } else {
      l_r[0] = __fadd_rn(l_r[0], __fadd_rn(p0, p1));
      l_r[1] = __fadd_rn(l_r[1], __fadd_rn(p2, p3));
    }
    s[4 * n] = p0; s[4 * n + 1] = p1; s[4 * n + 2] = p2; s[4 * n + 3] = p3;
  }
}

// One CTA per (BQ-row query tile, head, sample).  Warpgroup 0 (one lane) loads the Q tile once and streams K/V tiles
// of 64 keys through a TMA + mbarrier ring; warpgroups 1 .. CW each own 64 query rows: S = Q K^T (wgmma, both operands
// from shared memory, ceil(d / 16) k-steps), online softmax on the S registers (log2 domain), O += P V (wgmma with P as
// the register A operand and V read MN-major from shared memory: no transposed copy), then O / l -> fp16.  Keys past L
// arrive as zeros (TMA out-of-bounds fill of the per-head slab) and are masked to -inf in the last tile's softmax.
//
// Each consumer warpgroup runs a two-tile software pipeline: S_{j} = Q K_j^T and O += P_{j-1} V_{j-1} are issued as
// two commit groups, the softmax of tile j runs once the first retires (wait_group 1) while P V is still on the tensor
// cores, and O is rescaled by tile j's alpha after the second retires.  O therefore sees the same sequence of roundings
// as a serial loop: O_j = O_{j-1} * alpha_j + P_j V_j.  The stage of tile j-1 is released once its P V has retired.
// The consumer warpgroups take turns at issuing their MMAs (named barriers 1 .. CW, round robin), so that the MMAs of
// one run on the tensor cores while the others are in their softmax.
// DL (device length): the buffers hold p.L rows per head and sample, of which the first *p.len_dev are the sequence.  Query
// tiles at or past it exit, and only keys below it take part, masked in the last tile exactly as keys past p.L are.
//
// Shared calls (FaParams::period): CTA z serves frame f = z / groups and its inputs j0 .. j0 + G - 1, j0 = G (z mod
// groups), i.e. the samples f + j period that all have the attention map of sample f.  At G > 1 each stage holds K of
// sample f and the V tiles of the G samples; S and the softmax are computed once and each sample's O_g += P V_g is one
// wgmma per 16-key step, with the same shape as at G = 1, so every output element sees the same roundings as in the CTA
// of its own sample.  Inputs past the last (the last group of a ragged split) read the V of the frame's last input and
// write nothing.  With period 1 this is the merged layout: samples G z .. G z + G - 1, clamped to B - 1.
template <int KS, int G, bool DL>
__global__ void __launch_bounds__(FaCfg<KS, G>::THREADS, 1)
flash_attn_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_k,
                  const __grid_constant__ CUtensorMap tm_v, const FaParams p) {
  using Cf = FaCfg<KS, G>;
  constexpr int DV = Cf::DV;
  constexpr int STAGES = Cf::STAGES;
  extern __shared__ uint8_t fa_smem[];
  const uint32_t base = (smem_u32(fa_smem) + 1023u) & ~1023u;   // 128-byte swizzle: 1024-byte aligned tiles
  const uint32_t sq = base;
  const uint32_t skv = base + Cf::Q_BYTES;
  const uint32_t bars = skv + STAGES * Cf::STAGE_BYTES;
  const uint32_t q_full = bars;
  auto kv_full = [&](int s) { return bars + 8u * (1 + s); };
  auto kv_empty = [&](int s) { return bars + 8u * (1 + STAGES + s); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
  const int q0 = blockIdx.x * Cf::BQ, h = blockIdx.y;
  const int f = blockIdx.z / p.groups;                       // frame: the sample whose q / k the CTA reads
  const int j0 = (blockIdx.z - f * p.groups) * G;            // first input of the CTA's group
  const int b0 = f + j0 * p.period;                          // its sample
  const int seq = DL ? __ldg(p.len_dev) : p.L;               // keys that take part
  const int q_valid = DL ? seq : p.Lq;                       // query rows that are written
  if (DL && q0 >= q_valid) return;
  const int sqk = f * p.H + h;                               // slab of q / k
  const int nkv = (seq + FA_BKV - 1) / FA_BKV;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_q);
    tma_prefetch_desc(&tm_k);
    tma_prefetch_desc(&tm_v);
    mbar_init(q_full, 1);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(kv_full(s), 1);
      mbar_init(kv_empty(s), 4 * Cf::CW);                     // one arrival per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ===================== TMA producer =====================
    if constexpr (fa_moves_registers(KS)) setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(q_full, Cf::Q_BYTES);
      for (int a = 0; a < Cf::ATOMS; ++a) tma_load_3d(sq + a * Cf::Q_ATOM, &tm_q, q_full, 64 * a, q0, sqk);
      int stage = 0;
      uint32_t phase = 0;
      for (int j = 0; j < nkv; ++j) {
        mbar_wait(kv_empty(stage), phase ^ 1u);
        const uint32_t st = skv + stage * Cf::STAGE_BYTES;
        mbar_arrive_expect_tx(kv_full(stage), Cf::STAGE_BYTES);
        for (int a = 0; a < Cf::ATOMS; ++a) {
          tma_load_3d(st + a * Cf::KV_ATOM, &tm_k, kv_full(stage), 64 * a, j * FA_BKV, sqk);
          for (int g = 0; g < G; ++g) {
            const int sv = (G == 1 ? b0 : f + min(j0 + g, p.inputs - 1) * p.period) * p.H + h;   // slab of v
            tma_load_3d(st + (1 + g) * Cf::TILE_BYTES + a * Cf::KV_ATOM, &tm_v, kv_full(stage), 64 * a, j * FA_BKV, sv);
          }
        }
        if (++stage == STAGES) { stage = 0; phase ^= 1u; }
      }
    }
    return;
  }

  // ===================== consumers: 64 query rows per warpgroup =====================
  if constexpr (fa_moves_registers(KS)) setmaxnreg_inc<232>();
  const int cg = wg - 1, wq = warp & 3;
  float o[G][DV / 2];
#pragma unroll
  for (int g = 0; g < G; ++g)
#pragma unroll
    for (int i = 0; i < DV / 2; ++i) o[g][i] = 0.f;
  float m_r[2] = {-INFINITY, -INFINITY}, l_r[2] = {0.f, 0.f};   // rows 16 wq + lane/4 and + 8 of the warpgroup's 64
  float s[32], alpha[2];
  uint32_t pa[4][4];                                            // P as the register A operand of the four 16-key steps
  const uint32_t qa = sq + cg * 64 * 128;

  auto issue_qk = [&](int st) {
    const uint32_t kt = skv + st * Cf::STAGE_BYTES;
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
      const uint32_t off = (ks & 3) * 32u;   // k-step within the 64-column atom
      wgmma_m64n64k16_f16(s, wgmma_desc_sw128_kmajor(qa + (ks >> 2) * Cf::Q_ATOM + off),
                          wgmma_desc_sw128_kmajor(kt + (ks >> 2) * Cf::KV_ATOM + off), ks != 0 ? 1u : 0u);
    }
    wgmma_commit();
  };
  auto issue_pv = [&](int st) {
#pragma unroll
    for (int g = 0; g < G; ++g) {
      const uint32_t vt = skv + st * Cf::STAGE_BYTES + (1 + g) * Cf::TILE_BYTES;
#pragma unroll
      for (int kb = 0; kb < 4; ++kb)              // 16 keys per step: +16 rows x 128 B of the V tile
        wgmma_rs_f16_bt<DV>(o[g], pa[kb], wgmma_desc_sw128_mnmajor(vt + kb * 2048u, Cf::KV_ATOM), 1u);
    }
    wgmma_commit();
  };
  auto fence_s = [&]() {
#pragma unroll
    for (int i = 0; i < 32; ++i) reg_fence(s[i]);
  };
  auto fence_o = [&]() {
#pragma unroll
    for (int g = 0; g < G; ++g)
#pragma unroll
      for (int i = 0; i < DV / 2; ++i) reg_fence(o[g][i]);
  };
  auto pack_p = [&]() {
#pragma unroll
    for (int n = 0; n < 8; ++n) {
      pa[n >> 1][(n & 1) * 2] = pack_f16x2(s[4 * n], s[4 * n + 1]);
      pa[n >> 1][(n & 1) * 2 + 1] = pack_f16x2(s[4 * n + 2], s[4 * n + 3]);
    }
  };
  auto softmax = [&](int j) {
    if (j == nkv - 1) fa_softmax<true>(s, m_r, l_r, alpha, p.scale_log2, seq - j * FA_BKV, lane);
    else fa_softmax<false>(s, m_r, l_r, alpha, p.scale_log2, FA_BKV, lane);
  };
  auto release = [&](int st) {
    __syncwarp();
    if (lane == 0) mbar_arrive(kv_empty(st));     // this warp's MMAs on the stage have retired
  };
  // Issue turns: warpgroup cg waits on barrier 1 + cg and hands the turn to the next by arriving on its barrier.  Every
  // warpgroup issues nkv + 1 times; the last one grants warpgroup 0's first turn up front and skips its last hand-over,
  // so each barrier sees exactly as many arrivals as syncs.
  const int turns = nkv + 1;
  if (cg == Cf::CW - 1) bar_arrive_named(1, 256);
  auto turn_begin = [&]() { bar_sync_named(1 + cg, 256); };
  auto turn_end = [&](int t) {
    if (cg != Cf::CW - 1 || t + 1 < turns) bar_arrive_named(1 + (cg + 1) % Cf::CW, 256);
  };

  mbar_wait(q_full, 0);
  // tile 0: S only (O is still zero, so its rescale is skipped: 0 * alpha = 0)
  mbar_wait(kv_full(0), 0);
  turn_begin();
  wgmma_fence();
  issue_qk(0);
  turn_end(0);
  wgmma_wait<0>();
  fence_s();
  softmax(0);
  pack_p();
  int prev = 0, stage = 1;
  uint32_t phase = 0;
  if (stage == STAGES) { stage = 0; phase ^= 1u; }
  for (int j = 1; j < nkv; ++j) {
    mbar_wait(kv_full(stage), phase);
    turn_begin();
    wgmma_fence();
    issue_qk(stage);
    issue_pv(prev);
    turn_end(j);
    wgmma_wait<1>();                              // S_j has retired; P_{j-1} V_{j-1} may still run
    fence_s();
    softmax(j);
    wgmma_wait<0>();
    fence_o();
    release(prev);
#pragma unroll
    for (int g = 0; g < G; ++g)
#pragma unroll
      for (int n = 0; n < DV / 8; ++n) {
        o[g][4 * n] *= alpha[0]; o[g][4 * n + 1] *= alpha[0];
        o[g][4 * n + 2] *= alpha[1]; o[g][4 * n + 3] *= alpha[1];
      }
    pack_p();
    prev = stage;
    if (++stage == STAGES) { stage = 0; phase ^= 1u; }
  }
  // P V of the last tile
  turn_begin();
  wgmma_fence();
  issue_pv(prev);
  turn_end(nkv);
  wgmma_wait<0>();
  fence_o();
  release(prev);

  // O / l -> fp16, columns < head_dim
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    float l = l_r[r];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    // l = 0 only when every key of the row scored -inf: O = 0 then, as torch's attention and FlashAttention-2 return
    // (IEEE's 0 / 0 would be NaN); a NaN l still gives NaN
    const float inv = l == 0.f ? 1.f : 1.f / l;
    const int row = q0 + cg * 64 + wq * 16 + (lane >> 2) + 8 * r;
    if (row >= q_valid) continue;
#pragma unroll
    for (int g = 0; g < G; ++g) {
      if (G > 1 && j0 + g >= p.inputs) break;
      __half* dst = p.o + (static_cast<size_t>(b0 + g * p.period) * p.Lq + row) * p.C + h * p.d;
#pragma unroll
      for (int n = 0; n < DV / 8; ++n) {
        const int col = n * 8 + 2 * (lane & 3);
        if (col < p.d)
          *reinterpret_cast<uint32_t*>(dst + col) = pack_f16x2(o[g][4 * n + 2 * r] * inv, o[g][4 * n + 2 * r + 1] * inv);
      }
    }
  }
}

template <int KS, int G, bool DL>
int launch_fa(const __half* qh, const __half* kh, const __half* vh, __half* o, int B, int Lq, int L, int C, int H,
              int DP, float scale, int qk_period, cudaStream_t stream, const int* len_dev) {
  using Cf = FaCfg<KS, G>;
  if (H > 65535 || B > 65535 || Cf::ATOMS * 64 > DP) return VTM_E_SHAPE;
  if (G > 1 && !qk_period) return VTM_E_UNSUPPORTED;
  const int period = qk_period ? qk_period : B;               // not shared: every sample is a frame of its own
  if (period < 1 || B % period != 0) return VTM_E_SHAPE;
  const int inputs = B / period, groups = (inputs + G - 1) / G;
  constexpr int BQ = Cf::BQ;
  const uint64_t BH = static_cast<uint64_t>(B) * H;
  CUtensorMap tq, tk, tv;
  int rc = make_tmap_3d_f16(&tq, qh, DP, Lq, BH, DP, static_cast<uint64_t>(Lq) * DP, 64, BQ);
  if (rc) return rc;
  rc = make_tmap_3d_f16(&tk, kh, DP, L, BH, DP, static_cast<uint64_t>(L) * DP, 64, FA_BKV);
  if (rc) return rc;
  rc = make_tmap_3d_f16(&tv, vh, DP, L, BH, DP, static_cast<uint64_t>(L) * DP, 64, FA_BKV);
  if (rc) return rc;
  // shared-memory opt-in: once per instantiation and device (immutable afterwards)
  static bool opted[64];
  int dev = 0;
  rc = cuda_rc(cudaGetDevice(&dev));
  if (rc) return rc;
  if (dev < 0 || dev >= 64 || !opted[dev]) {
    rc = cuda_rc(cudaFuncSetAttribute(flash_attn_kernel<KS, G, DL>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      static_cast<int>(Cf::SMEM_BYTES)));
    if (rc) return rc;
    if (dev >= 0 && dev < 64) opted[dev] = true;
  }
  FaParams p;
  p.o = o;
  p.L = L; p.Lq = Lq; p.H = H; p.d = C / H; p.C = C; p.B = B;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.period = period; p.inputs = inputs; p.groups = groups;
  p.len_dev = len_dev;
  const dim3 grid(static_cast<unsigned>((Lq + BQ - 1) / BQ), static_cast<unsigned>(H),
                  static_cast<unsigned>(period * groups));
  flash_attn_kernel<KS, G, DL><<<grid, Cf::THREADS, Cf::SMEM_BYTES, stream>>>(tq, tk, tv, p);
  return launch_rc();
}

// launch_fa<KS, g, DL> for a run-time group size 1 <= g <= G
template <int KS, int G, bool DL>
int launch_fa_group(int g, const __half* qh, const __half* kh, const __half* vh, __half* o, int B, int Lq, int L, int C,
                    int H, int DP, float scale, int qk_period, cudaStream_t stream, const int* len_dev) {
  if constexpr (G > 1) {
    if (g < G) return launch_fa_group<KS, G - 1, DL>(g, qh, kh, vh, o, B, Lq, L, C, H, DP, scale, qk_period, stream, len_dev);
  }
  return launch_fa<KS, G, DL>(qh, kh, vh, o, B, Lq, L, C, H, DP, scale, qk_period, stream, len_dev);
}

// Samples per CTA: 1, or for a shared call the fewest groups of at most fa_group_max(KS) of a frame's `inputs` samples,
// equally sized (so that the last group reads as few clamped V tiles as possible).
inline int fa_group(int KS, int inputs, int qk_period) {
  if (!qk_period) return 1;
  const int gmax = fa_group_max(KS);
  const int groups = (inputs + gmax - 1) / gmax;
  return (inputs + groups - 1) / groups;
}

// qk_period: 0 (not shared), or n >= 1 with B % n == 0: sample b reads the q / k slab of sample b mod n (FaParams).
int launch_fa_any(const __half* qh, const __half* kh, const __half* vh, __half* o, int B, int Lq, int L, int C, int H,
                  int DP, float scale, int qk_period, cudaStream_t stream, const int* len_dev = nullptr) {
  if (qk_period < 0 || (qk_period && B % qk_period != 0)) return VTM_E_SHAPE;
  const int ks = (C / H + 15) / 16;
  const int g = fa_group(ks, qk_period ? B / qk_period : 1, qk_period);
#define VTM_FA_CASE(KS)                                                                                               \
  case KS:                                                                                                            \
    return len_dev ? launch_fa_group<KS, fa_group_max(KS), true>(g, qh, kh, vh, o, B, Lq, L, C, H, DP, scale,         \
                                                                 qk_period, stream, len_dev)                         \
                   : launch_fa_group<KS, fa_group_max(KS), false>(g, qh, kh, vh, o, B, Lq, L, C, H, DP, scale,        \
                                                                  qk_period, stream, nullptr);
  if (C / H > FA_MAX_HEAD_DIM) return VTM_E_UNSUPPORTED;
  switch (ks) {
    VTM_FA_CASE(1)
    VTM_FA_CASE(2)
    VTM_FA_CASE(3)
    VTM_FA_CASE(4)
    VTM_FA_CASE(5)
    VTM_FA_CASE(6)
    VTM_FA_CASE(7)
    VTM_FA_CASE(8)
    VTM_FA_CASE(9)
    VTM_FA_CASE(10)
    default:
      return VTM_E_UNSUPPORTED;
  }
#undef VTM_FA_CASE
}

}  // namespace
}  // namespace vtm

extern "C" size_t vtm_attention_workspace_bytes(int32_t B, int32_t L, int32_t C, int32_t heads) {
  (void)heads;
  if (B <= 0 || L <= 0 || C <= 0) return 0;
  if (heads <= 0 || C % heads != 0) return 0;
  const size_t DP = vtm::fa_padded_row(C / heads);
  // q/k/v head-major [3][B][H][L][DP] + o [B*L, C], fp16
  return (static_cast<size_t>(3) * B * heads * L * DP + static_cast<size_t>(B) * L * C) * 2 + 256;
}

extern "C" size_t vtm_attention_lora_workspace_bytes(int32_t B, int32_t L, int32_t C, int32_t heads, int32_t R_qkv,
                                                     int32_t R_o) {
  const size_t base = vtm_attention_workspace_bytes(B, L, C, heads);
  if (base == 0 || R_qkv < 0 || R_o < 0) return 0;
  // T of the QKV GEMM, then of the output projection, in one [B*L, max(R_qkv, R_o)] buffer after o
  return base + static_cast<size_t>(B) * L * (R_qkv > R_o ? R_qkv : R_o) * 2;
}

namespace vtm {
namespace {
// len_dev: NULL, or the sequence length on the device with L the rows of the buffers (vtm_attention_dev).
// qk_items (VTM_ATTN_SHARED_QK only): sample b reads the queries and keys of sample b mod qk_items (1 <= qk_items,
// B % qk_items == 0).
int attention_impl(const void* x_dev, const void* w_qkv_dev, const void* w_o_dev, const void* b_o_dev, int32_t B,
                   int32_t L, int32_t C, int32_t heads, float scale, int32_t flags, const int32_t* len_dev, void* y_dev,
                   void* ws_dev, size_t ws_bytes, void* stream_, const vtm_lora_t* lora_qkv = nullptr,
                   const vtm_lora_t* lora_o = nullptr, const void* resid_dev = nullptr, int32_t qk_items = 1) {
  if (!x_dev || !w_qkv_dev || !w_o_dev || !y_dev || !ws_dev) return VTM_E_NULL;
  if (B <= 0 || L <= 0 || C <= 0 || heads <= 0 || C % heads != 0) return VTM_E_SHAPE;
  const int d = C / heads;
  if (d % 8 != 0 || C % 8 != 0) return VTM_E_SHAPE;
  if (d > FA_MAX_HEAD_DIM || (flags & ~1) != 0) return VTM_E_UNSUPPORTED;
  const int period = (flags & 1) ? qk_items : 0;             // launch_fa_any's qk_period
  if ((flags & 1) && (qk_items < 1 || B % qk_items != 0)) return VTM_E_SHAPE;
  int Rq = 0, Ro = 0;
  int rc = lora_rank(lora_qkv, &Rq);
  if (rc) return rc;
  rc = lora_rank(lora_o, &Ro);
  if (rc) return rc;
  if (ws_bytes < vtm_attention_lora_workspace_bytes(B, L, C, heads, Rq, Ro)) return VTM_E_WS;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int DP = fa_padded_row(d);
  __half* qkv = static_cast<__half*>(ws_dev);
  __half* o = qkv + static_cast<size_t>(3) * B * heads * L * DP;
  const int M = B * L;
  const size_t slab = static_cast<size_t>(B) * heads * L * DP;    // one of q, k, v for all samples
  __half* kh = qkv + slab;
  __half* vh = kh + slab;
  __half* t = o + static_cast<size_t>(M) * C;                      // LoRA T buffer [M, max(Rq, Ro)]
  const __half* uq = Rq ? static_cast<const __half*>(lora_qkv->up_dev) : nullptr;
  if (Rq) {
    rc = vtm_linear_f16(x_dev, lora_qkv->down_dev, nullptr, M, Rq, C, t, Rq, stream_);
    if (rc) return rc;
  }
  if (flags & 1) {
    // shared: q and k of samples 0 .. qk_items - 1 (the only ones the flash kernel reads: their first qk_items L rows of
    // x and of T), v of every sample
    rc = launch_head_proj(x_dev, w_qkv_dev, qkv, qk_items, L, C, C, heads, DP, 0, 2, stream,
                          static_cast<long long>(slab), t, uq, Rq);
    if (rc) return rc;
    rc = launch_head_proj(x_dev, static_cast<const __half*>(w_qkv_dev) + static_cast<size_t>(2) * C * C, vh, B, L, C, C,
                          heads, DP, 2, 1, stream, 0, t, Rq ? uq + static_cast<size_t>(2) * C * Rq : nullptr, Rq);
  } else {
    rc = launch_head_proj(x_dev, w_qkv_dev, qkv, B, L, C, C, heads, DP, 0, 3, stream, 0, t, uq, Rq);
  }
  if (rc) return rc;
  rc = launch_fa_any(qkv, kh, vh, o, B, L, L, C, heads, DP, scale, period, stream, len_dev);
  if (rc) return rc;
  if (Ro)
    return vtm_linear_lora_f16(o, w_o_dev, b_o_dev, resid_dev, resid_dev ? C : 0, lora_o, M, C, C, y_dev, C, t,
                               static_cast<size_t>(M) * Ro * 2, stream_);
  if (resid_dev) return vtm_linear_residual_f16(o, w_o_dev, b_o_dev, resid_dev, C, M, C, C, y_dev, C, stream_);
  return vtm_linear_f16(o, w_o_dev, b_o_dev, M, C, C, y_dev, C, stream_);
}
}  // namespace
}  // namespace vtm

extern "C" int vtm_attention_ex(const void* x_dev, const void* w_qkv_dev, const void* w_o_dev, const void* b_o_dev,
                                int32_t B, int32_t L, int32_t C, int32_t heads, float scale, int32_t flags, void* y_dev,
                                void* ws_dev, size_t ws_bytes, void* stream_) {
  return vtm::attention_impl(x_dev, w_qkv_dev, w_o_dev, b_o_dev, B, L, C, heads, scale, flags, nullptr, y_dev, ws_dev,
                             ws_bytes, stream_);
}

extern "C" int vtm_attention_dev(const void* x_dev, const void* w_qkv_dev, const void* w_o_dev, const void* b_o_dev,
                                 int32_t B, int32_t L_cap, int32_t C, int32_t heads, float scale, int32_t flags,
                                 const int32_t* len_dev, void* y_dev, void* ws_dev, size_t ws_bytes, void* stream_) {
  if (!len_dev) return VTM_E_NULL;
  return vtm::attention_impl(x_dev, w_qkv_dev, w_o_dev, b_o_dev, B, L_cap, C, heads, scale, flags, len_dev, y_dev,
                             ws_dev, ws_bytes, stream_);
}

extern "C" int vtm_attention_lora(const void* x_dev, const void* w_qkv_dev, const void* w_o_dev, const void* b_o_dev,
                                  const vtm_lora_t* lora_qkv, const vtm_lora_t* lora_o, int32_t B, int32_t L, int32_t C,
                                  int32_t heads, float scale, int32_t flags, const int32_t* len_dev, void* y_dev,
                                  void* ws_dev, size_t ws_bytes, void* stream_) {
  return vtm::attention_impl(x_dev, w_qkv_dev, w_o_dev, b_o_dev, B, L, C, heads, scale, flags, len_dev, y_dev, ws_dev,
                             ws_bytes, stream_, lora_qkv, lora_o);
}

// Self-attention of an unmerged block with its residual: attn1(norm1(h)) + h (vidtome/patch.py:157-169 with u = m =
// do_nothing), the residual added in the out projection's epilogue as vtm_linear_residual_f16 does.
extern "C" int vtm_attention_residual(const void* x_dev, const void* w_qkv_dev, const void* w_o_dev,
                                      const void* b_o_dev, const void* resid_dev, const vtm_lora_t* lora_qkv,
                                      const vtm_lora_t* lora_o, int32_t B, int32_t L, int32_t C, int32_t heads,
                                      float scale, void* y_dev, void* ws_dev, size_t ws_bytes, void* stream_) {
  if (!resid_dev) return VTM_E_NULL;
  return vtm::attention_impl(x_dev, w_qkv_dev, w_o_dev, b_o_dev, B, L, C, heads, scale, 0, nullptr, y_dev, ws_dev,
                             ws_bytes, stream_, lora_qkv, lora_o, resid_dev);
}

// The same with PnP's injection over the frames of an unmerged block (utils/pnp_utils.py:57-68,86-91): under
// VTM_ATTN_SHARED_QK the batch is [source | uncond | cond] runs of qk_items frames, and item b uses the attention map
// of item b mod qk_items.
extern "C" int vtm_attention_residual_ex(const void* x_dev, const void* w_qkv_dev, const void* w_o_dev,
                                         const void* b_o_dev, const void* resid_dev, const vtm_lora_t* lora_qkv,
                                         const vtm_lora_t* lora_o, int32_t B, int32_t L, int32_t C, int32_t heads,
                                         float scale, int32_t flags, int32_t qk_items, void* y_dev, void* ws_dev,
                                         size_t ws_bytes, void* stream_) {
  if (!resid_dev) return VTM_E_NULL;
  return vtm::attention_impl(x_dev, w_qkv_dev, w_o_dev, b_o_dev, B, L, C, heads, scale, flags, nullptr, y_dev, ws_dev,
                             ws_bytes, stream_, lora_qkv, lora_o, resid_dev, qk_items);
}

extern "C" int vtm_attention(const void* x_dev, const void* w_qkv_dev, const void* w_o_dev, const void* b_o_dev,
                             int32_t B, int32_t L, int32_t C, int32_t heads, float scale, void* y_dev,
                             void* ws_dev, size_t ws_bytes, void* stream_) {
  return vtm_attention_ex(x_dev, w_qkv_dev, w_o_dev, b_o_dev, B, L, C, heads, scale, 0, y_dev, ws_dev, ws_bytes, stream_);
}

// ------------------------------------------------------------------------------------------------------------------
// Cross-attention of the patched block (vidtome/patch.py:171-185: `self.attn2(norm2(h), encoder_hidden_states=ctx)` and
// the residual add) — diffusers Attention with K/V from the text context.
extern "C" size_t vtm_cross_attention_workspace_bytes(int32_t B, int32_t Lq, int32_t Lk, int32_t C, int32_t heads) {
  if (B <= 0 || Lq <= 0 || Lk <= 0 || C <= 0 || heads <= 0 || C % heads != 0) return 0;
  const size_t DP = vtm::fa_padded_row(C / heads);
  return (static_cast<size_t>(B) * heads * (static_cast<size_t>(Lq) + 2 * static_cast<size_t>(Lk)) * DP +
          static_cast<size_t>(B) * Lq * C) * 2 + 512;
}

extern "C" size_t vtm_cross_attention_lora_workspace_bytes(int32_t B, int32_t Lq, int32_t Lk, int32_t C, int32_t heads,
                                                           int32_t R_q, int32_t R_kv, int32_t R_o) {
  const size_t base = vtm_cross_attention_workspace_bytes(B, Lq, Lk, C, heads);
  if (base == 0 || R_q < 0 || R_kv < 0 || R_o < 0) return 0;
  // T of to_q, then of to_out, in one [B*Lq, max(R_q, R_o)] buffer; T of to_k / to_v [B*Lk, R_kv]
  return base + (static_cast<size_t>(B) * Lq * (R_q > R_o ? R_q : R_o) + static_cast<size_t>(B) * Lk * R_kv) * 2;
}

namespace vtm {
namespace {
int cross_attention_impl(const void* x_dev, const void* ctx_dev, const void* w_q_dev, const void* w_kv_dev,
                         const void* w_o_dev, const void* b_o_dev, const void* resid_dev, const vtm_lora_t* lora_q,
                         const vtm_lora_t* lora_kv, const vtm_lora_t* lora_o, int32_t B, int32_t Lq, int32_t Lk,
                         int32_t C, int32_t Cctx, int32_t heads, float scale, void* y_dev, void* ws_dev, size_t ws_bytes,
                         void* stream_) {
  if (!x_dev || !ctx_dev || !w_q_dev || !w_kv_dev || !w_o_dev || !y_dev || !ws_dev) return VTM_E_NULL;
  if (B <= 0 || Lq <= 0 || Lk <= 0 || C <= 0 || Cctx <= 0 || heads <= 0 || C % heads != 0) return VTM_E_SHAPE;
  const int d = C / heads;
  if (d % 8 != 0 || C % 8 != 0 || Cctx % 8 != 0) return VTM_E_SHAPE;
  if (d > FA_MAX_HEAD_DIM) return VTM_E_UNSUPPORTED;
  int Rq = 0, Rkv = 0, Ro = 0;
  int rc = lora_rank(lora_q, &Rq);
  if (rc) return rc;
  rc = lora_rank(lora_kv, &Rkv);
  if (rc) return rc;
  rc = lora_rank(lora_o, &Ro);
  if (rc) return rc;
  if (ws_bytes < vtm_cross_attention_lora_workspace_bytes(B, Lq, Lk, C, heads, Rq, Rkv, Ro)) return VTM_E_WS;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int DP = fa_padded_row(d);
  __half* qh = static_cast<__half*>(ws_dev);
  __half* kh = qh + static_cast<size_t>(B) * heads * Lq * DP;
  __half* vh = kh + static_cast<size_t>(B) * heads * Lk * DP;
  __half* o = vh + static_cast<size_t>(B) * heads * Lk * DP;
  const int M = B * Lq;
  __half* tq = o + static_cast<size_t>(M) * C;                      // T of to_q / to_out [M, max(Rq, Ro)]
  __half* tkv = tq + static_cast<size_t>(M) * (Rq > Ro ? Rq : Ro);  // T of to_k / to_v [B * Lk, Rkv]
  if (Rq) {
    rc = vtm_linear_f16(x_dev, lora_q->down_dev, nullptr, M, Rq, C, tq, Rq, stream_);
    if (rc) return rc;
  }
  rc = launch_head_proj(x_dev, w_q_dev, qh, B, Lq, C, C, heads, DP, 0, 1, stream, 0, tq, Rq ? lora_q->up_dev : nullptr,
                        Rq);
  if (rc) return rc;
  if (Rkv) {
    rc = vtm_linear_f16(ctx_dev, lora_kv->down_dev, nullptr, B * Lk, Rkv, Cctx, tkv, Rkv, stream_);
    if (rc) return rc;
  }
  rc = launch_head_proj(ctx_dev, w_kv_dev, kh, B, Lk, Cctx, C, heads, DP, 1, 2, stream, 0, tkv,
                        Rkv ? lora_kv->up_dev : nullptr, Rkv);
  if (rc) return rc;
  rc = launch_fa_any(qh, kh, vh, o, B, Lq, Lk, C, heads, DP, scale, 0, stream);
  if (rc) return rc;
  if (Ro)
    return vtm_linear_lora_f16(o, w_o_dev, b_o_dev, resid_dev, C, lora_o, M, C, C, y_dev, C, tq,
                               static_cast<size_t>(M) * Ro * 2, stream_);
  if (resid_dev) return vtm_linear_residual_f16(o, w_o_dev, b_o_dev, resid_dev, C, M, C, C, y_dev, C, stream_);
  return vtm_linear_f16(o, w_o_dev, b_o_dev, M, C, C, y_dev, C, stream_);
}
}  // namespace
}  // namespace vtm

extern "C" int vtm_cross_attention(const void* x_dev, const void* ctx_dev, const void* w_q_dev, const void* w_kv_dev,
                                   const void* w_o_dev, const void* b_o_dev, const void* resid_dev, int32_t B, int32_t Lq,
                                   int32_t Lk, int32_t C, int32_t Cctx, int32_t heads, float scale, void* y_dev,
                                   void* ws_dev, size_t ws_bytes, void* stream_) {
  return vtm::cross_attention_impl(x_dev, ctx_dev, w_q_dev, w_kv_dev, w_o_dev, b_o_dev, resid_dev, nullptr, nullptr,
                                   nullptr, B, Lq, Lk, C, Cctx, heads, scale, y_dev, ws_dev, ws_bytes, stream_);
}

extern "C" int vtm_cross_attention_lora(const void* x_dev, const void* ctx_dev, const void* w_q_dev,
                                        const void* w_kv_dev, const void* w_o_dev, const void* b_o_dev,
                                        const void* resid_dev, const vtm_lora_t* lora_q, const vtm_lora_t* lora_kv,
                                        const vtm_lora_t* lora_o, int32_t B, int32_t Lq, int32_t Lk, int32_t C,
                                        int32_t Cctx, int32_t heads, float scale, void* y_dev, void* ws_dev,
                                        size_t ws_bytes, void* stream_) {
  return vtm::cross_attention_impl(x_dev, ctx_dev, w_q_dev, w_kv_dev, w_o_dev, b_o_dev, resid_dev, lora_q, lora_kv,
                                   lora_o, B, Lq, Lk, C, Cctx, heads, scale, y_dev, ws_dev, ws_bytes, stream_);
}
