// KA — fused cosine-similarity GEMM + row arg-max for sm_90a.
//
// Reference semantics (vidtome/merge.py:87,112 / :392,416 and the align_batch variant :93-97):
//   scores = a @ b^T            (fp16 result: fp32 accumulate, round-to-nearest-even to fp16)
//   node_max, node_idx = scores.max(-1)   (first index among equal maxima)
// Here the Ns x Nd score matrix never exists.  Each CTA takes a work item = (128-row block of src tokens, sample,
// range of 256-token dst tiles), computes every 128 x 256 score tile with wgmma into registers and keeps, per src row,
// a running (max, first arg) straight from the accumulator fragments.  Partial results are merged across dst ranges /
// samples with a 64-bit atomicMax on a packed (ordered score, ~arg) key, which realises exactly "largest score, then
// smallest index".
//
// Kernel layout (persistent grid, 384 threads = three warpgroups):
//   warpgroup 0      TMA producer (one lane issues);
//   warpgroups 1, 2  wgmma m64n256k16 consumers, each owning 64 src rows of the tile (128 fp32 accumulators/thread).
// Shared memory, resident-A form (the work item's whole 128 x C src block fits next to >= 3 ring stages within 227 KB:
// C <= 512, with 6 dst stages up to C = 128, 5 up to 256, 4 up to 384 and 3 up to 512): the src block stays in shared memory for the whole work item, one 128B-swizzled 64-column chunk
// per K step, each guarded by its own full/empty mbarrier pair, and the ring carries only dst tiles (256 x 64).  A
// chunk is refilled for the next work item as soon as the last tile's wgmma on it has retired, so the producer keeps
// running ahead across work items.  Per dst tile only the dst bytes come from L2: 128 FLOP per byte instead of 64 for
// a ring that carries both operands.
// Streaming-A form (larger C): every ring stage carries the src chunk too, as in a plain GEMM mainloop.
#include <stdlib.h>

#include "common.cuh"
#include "ptx.cuh"

namespace vtm {
namespace {

namespace ka {
constexpr int BM = 128;
constexpr int BN = 256;
constexpr int BK = 64;
constexpr int UK = 16;
constexpr int CONSUMER_WARPS = 8;
constexpr int THREADS = 384;
constexpr uint32_t A_BYTES = BM * BK * 2;   // one src chunk: 16 KB
constexpr uint32_t B_BYTES = BN * BK * 2;   // one dst chunk: 32 KB
constexpr int MAX_STAGES = 6;
constexpr int MIN_RESIDENT_STAGES = 3;      // fewer ring stages than this starve the tensor cores
constexpr int MAX_A_CHUNKS = 8;
constexpr size_t SMEM_LIMIT = 227 * 1024;   // opt-in shared memory per block on sm_90
// 1024 B of alignment slack + 8-byte barrier slots: full[MAX_STAGES] | empty[MAX_STAGES] | a_full[..] | a_empty[..]
constexpr uint32_t BAR_BYTES = 8u * (2 * MAX_STAGES + 2 * MAX_A_CHUNKS);
constexpr size_t FIXED = 1024 + BAR_BYTES;
// Work items per SM the dst sweep is split into (when the problem allows).  Each item costs one src-block load and one
// atomic per src row; finer items balance the persistent grid.  At ds1 level 1 (49152 x 16384 x 320, B = 2) on an H100
// 80GB HBM3 at 400 W, 4, 8 and 16 items per SM timed within 2 % of each other; 8 was the fastest.
constexpr int TARGET_ITEMS_PER_SM = 8;

// Shared-memory layout chosen from C on the host: resident src block when it fits with MIN_RESIDENT_STAGES dst stages.
struct Layout {
  int resident;
  int stages;
  uint32_t stage_bytes;
  uint32_t a_bytes;   // resident src block (0 when streaming)
  __host__ void plan(int k_chunks) {
    const size_t a_res = static_cast<size_t>(k_chunks) * A_BYTES;
    resident = k_chunks <= MAX_A_CHUNKS && FIXED + a_res + MIN_RESIDENT_STAGES * B_BYTES <= SMEM_LIMIT;
    a_bytes = resident ? static_cast<uint32_t>(a_res) : 0u;
    stage_bytes = resident ? B_BYTES : A_BYTES + B_BYTES;
    const int fit = static_cast<int>((SMEM_LIMIT - FIXED - a_bytes) / stage_bytes);
    stages = fit > MAX_STAGES ? MAX_STAGES : fit;
  }
  __host__ size_t smem_bytes() const { return FIXED + a_bytes + static_cast<size_t>(stages) * stage_bytes; }
};

// Work item = (src block, b, [nt0, nt1)), src block fastest: the dst ranges of one src block run far apart in time, so
// a later range starts from the maxima the earlier ones published.
struct Items {
  int batches;
  int m_tiles, n_tiles, tiles_per_split, n_splits;
  int k_chunks;
  int total;
  __host__ void plan(int M, int N, int K, int B, int sms, int target_items_per_sm) {
    batches = B;
    m_tiles = (M + BM - 1) / BM;
    n_tiles = (N + BN - 1) / BN;
    k_chunks = (K + BK - 1) / BK;
    const long long base = static_cast<long long>(m_tiles) * B;
    int s = 1;
    while (base * s < static_cast<long long>(target_items_per_sm) * sms && s * 2 <= n_tiles) s *= 2;
    tiles_per_split = (n_tiles + s - 1) / s;
    n_splits = (n_tiles + tiles_per_split - 1) / tiles_per_split;
    total = static_cast<int>(base * n_splits);
  }
  __device__ __forceinline__ void decode(int w, int* m_tile, int* b, int* nt0, int* nt1) const {
    *m_tile = w % m_tiles;
    const int rest = w / m_tiles;
    *b = rest % batches;
    const int sp = rest / batches;
    *nt0 = sp * tiles_per_split;
    const int e = *nt0 + tiles_per_split;
    *nt1 = e < n_tiles ? e : n_tiles;
  }
};

struct Args {
  unsigned long long* keys;  // [B', ld]
  int Ns, Nd, align_batch;
  int ld;                    // row stride of keys: Ns, or the src capacity with device counts
  const int* counts;         // device counts {Ns, Nd, ...} (vtm_sim_argmax_dev), NULL = the values above
};

__device__ __forceinline__ float round_f16(float x) { return __half2float(__float2half_rn(x)); }

// Running (max, first arg) of one src row over this thread's columns.  A work item starts from what other items (other
// dst ranges / samples of the same src rows) have already published: scores below the published maximum cannot win, so
// they are filtered on group maxima and the per-element scan runs only for the rare group that holds a candidate.  The
// threshold is the fp16 value just BELOW the published maximum, so an equal score still becomes a candidate and the
// packed-key atomicMax resolves the tie towards the smaller dst index.  Any stale value read here is a valid (lower)
// threshold: published keys only grow.
struct RowBest {
  float best;          // running maximum, or the entry threshold while idx is "none"
  uint32_t idx;
  __device__ __forceinline__ void begin(const Args& p, int row, int b) {
    best = -INFINITY;
    idx = 0xFFFFFFFFu;
    if (row < p.Ns) {
      const size_t o = (p.align_batch ? 0 : static_cast<size_t>(b) * p.ld) + row;
      const unsigned long long k = *reinterpret_cast<const volatile unsigned long long*>(p.keys + o);
      uint32_t ord = static_cast<uint32_t>(k >> 32);
      if (k != 0ull && ord > 0x0400u) {          // published and above -inf
        ord -= 1u;
        if (ord == 0x7FFFu) ord = 0x7FFEu;       // below +0 comes -0, which compares equal: step once more
        best = __half2float(__ushort_as_half(static_cast<unsigned short>(ordered_to_half_bits(ord))));
      }
    }
  }
  // The four lanes of a quad hold disjoint columns of the row: "larger score, then smaller index" over the quad gives
  // the row's (max, first arg).  A lane without a candidate holds the common threshold, below any candidate.
  __device__ __forceinline__ void quad_reduce() {
#pragma unroll
    for (int o = 1; o <= 2; o <<= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const uint32_t oi = __shfl_xor_sync(0xffffffffu, idx, o);
      if (ob > best || (ob == best && oi < idx)) { best = ob; idx = oi; }
    }
  }
  __device__ __forceinline__ void publish(const Args& p, int row, int b) const {
    if (row < p.Ns && idx != 0xFFFFFFFFu) {
      const uint32_t hb = static_cast<uint32_t>(__half_as_ushort(__float2half_rn(best)));
      const uint32_t arg = p.align_batch ? static_cast<uint32_t>(b) * static_cast<uint32_t>(p.Nd) + idx : idx;
      const size_t o = (p.align_batch ? 0 : static_cast<size_t>(b) * p.ld) + row;
      atomicMax(p.keys + o, static_cast<unsigned long long>(pack_key(hb, arg)));
    }
  }
};

// Arg-max over one finished 64 x 256 accumulator tile of a warpgroup.  Fragment layout (m64nNk16): for n8 block j,
// d[4j + 2h + e] is row 16 w + l / 4 + 8 h, column 8 j + 2 (l % 4) + e.  A thread's columns of a row ascend with
// (j, e), so a strict '>' scan in that order keeps the first index among equals.
__device__ __forceinline__ void tile_argmax(const float (&d)[128], RowBest (&rb)[2], int col0, int Nd, int lane) {
  const int c_lane = 2 * (lane & 3);
  if (col0 + BN <= Nd) {
    // Rounding to fp16 is monotonic, so max(round(x_i)) == round(max(x_i)): filter on the fp32 maxima of four
    // 64-column groups (16 values per thread and row).  The branch is warp-wide, hence the fine groups.
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float g[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        float m0 = fmaxf(d[32 * q + 2 * h], d[32 * q + 2 * h + 1]);
        float m1 = fmaxf(d[32 * q + 4 + 2 * h], d[32 * q + 4 + 2 * h + 1]);
#pragma unroll
        for (int j = 2; j < 8; j += 2) {
          m0 = fmaxf(m0, fmaxf(d[32 * q + 4 * j + 2 * h], d[32 * q + 4 * j + 2 * h + 1]));
          m1 = fmaxf(m1, fmaxf(d[32 * q + 4 * (j + 1) + 2 * h], d[32 * q + 4 * (j + 1) + 2 * h + 1]));
        }
        g[q] = fmaxf(m0, m1);
      }
      if (round_f16(fmaxf(fmaxf(g[0], g[1]), fmaxf(g[2], g[3]))) > rb[h].best) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          if (round_f16(g[q]) > rb[h].best) {   // ascending groups and strict '>' keep the first index among equals
#pragma unroll
            for (int j = 8 * q; j < 8 * q + 8; ++j) {
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const float hv = round_f16(d[4 * j + 2 * h + e]);
                if (hv > rb[h].best) { rb[h].best = hv; rb[h].idx = static_cast<uint32_t>(col0 + 8 * j + c_lane + e); }
              }
            }
          }
        }
      }
    }
  } else {
    // last dst tile: columns >= Nd hold TMA zero fill and must not take part
    const int n_valid = Nd - col0 - c_lane;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
      for (int j = 0; j < 32; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float hv = round_f16(d[4 * j + 2 * h + e]);
          if (8 * j + e < n_valid && hv > rb[h].best) {
            rb[h].best = hv;
            rb[h].idx = static_cast<uint32_t>(col0 + 8 * j + c_lane + e);
          }
        }
      }
    }
  }
}

__global__ void __launch_bounds__(THREADS, 1)
sim_argmax_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                  const Items wk, const Layout lay, const Args p_in) {
  extern __shared__ uint8_t smem_raw[];
  // with device counts the grid is planned for capacity: src blocks at or past Ns and dst tiles at or past Nd are
  // skipped (by the producer and the consumers alike, so the barrier phases stay paired)
  Args p = p_in;
  if (p.counts) {
    p.Ns = __ldg(p.counts);
    p.Nd = __ldg(p.counts + 1);
  }
  const int nt_end = (p.Nd + BN - 1) / BN;
  // 1024-byte alignment: required by the 128-byte swizzle pattern shared by TMA and wgmma descriptors
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t a_base = smem_base;                   // resident src block: k_chunks x A_BYTES
  const uint32_t ring_base = smem_base + lay.a_bytes;  // stages x stage_bytes
  const uint32_t bar_base = ring_base + static_cast<uint32_t>(lay.stages) * lay.stage_bytes;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (MAX_STAGES + s); };
  auto a_full_bar = [&](int kc) { return bar_base + 8u * (2 * MAX_STAGES + kc); };
  auto a_empty_bar = [&](int kc) { return bar_base + 8u * (2 * MAX_STAGES + MAX_A_CHUNKS + kc); };
  const int stages = lay.stages;
  const bool resident = lay.resident != 0;
  // B (dst) data offset within a stage: after the src chunk in the streaming form
  const uint32_t b_off = resident ? 0u : A_BYTES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  // this CTA's work items: w_first, w_first + w_step, ...
  const int w_first = static_cast<int>(blockIdx.x);
  const int w_step = static_cast<int>(gridDim.x);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    for (int s = 0; s < stages; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), CONSUMER_WARPS);
    }
    if (resident) {
      for (int kc = 0; kc < wk.k_chunks; ++kc) {
        mbar_init(a_full_bar(kc), 1);
        mbar_init(a_empty_bar(kc), CONSUMER_WARPS);
      }
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0, a_phase = 0;
      const uint32_t stage_tx = lay.stage_bytes;   // src chunk (streaming) + dst chunk
      for (int w = w_first; w < wk.total; w += w_step) {
        int m_tile, b, nt0, nt1;
        wk.decode(w, &m_tile, &b, &nt0, &nt1);
        if (nt1 > nt_end) nt1 = nt_end;
        if (nt0 >= nt1 || m_tile * BM >= p.Ns) continue;
        for (int nt = nt0; nt < nt1; ++nt) {
          for (int kc = 0; kc < wk.k_chunks; ++kc) {
            if (resident && nt == nt0) {
              // chunk kc of the src block: free once the previous item's last tile has retired its wgmma on it
              mbar_wait(a_empty_bar(kc), a_phase ^ 1u);
              mbar_arrive_expect_tx(a_full_bar(kc), A_BYTES);
              tma_load_3d(a_base + kc * A_BYTES, &tmap_a, a_full_bar(kc), kc * BK, m_tile * BM, b);
            }
            const uint32_t sa = ring_base + stage * lay.stage_bytes;
            mbar_wait(empty_bar(stage), phase ^ 1u);
            mbar_arrive_expect_tx(full_bar(stage), stage_tx);
            if (!resident) tma_load_3d(sa, &tmap_a, full_bar(stage), kc * BK, m_tile * BM, b);
            tma_load_3d(sa + b_off, &tmap_b, full_bar(stage), kc * BK, nt * BN, b);
            if (++stage == stages) { stage = 0; phase ^= 1u; }
          }
        }
        a_phase ^= 1u;
      }
    }
  } else {
    // ===================== MMA + arg-max =====================
    setmaxnreg_inc<232>();
    const int cg = wg - 1;                        // which 64 rows of the tile
    const int wq = warp & 3;                      // warp within the warpgroup
    const int r0 = cg * 64 + wq * 16 + (lane >> 2);   // this thread's rows of the tile: r0 and r0 + 8
    int stage = 0;
    uint32_t phase = 0, a_phase = 0;
    float d[128];
    // smem slot reusable: this warp's MMAs reading it have retired
    auto release = [&](int st) {
      __syncwarp();
      if (lane == 0) mbar_arrive(empty_bar(st));
    };
    auto release_a = [&](int kc) {
      __syncwarp();
      if (lane == 0) mbar_arrive(a_empty_bar(kc));
    };
    for (int w = w_first; w < wk.total; w += w_step) {
      int m_tile, b, nt0, nt1;
      wk.decode(w, &m_tile, &b, &nt0, &nt1);
      if (nt1 > nt_end) nt1 = nt_end;
      if (nt0 >= nt1 || m_tile * BM >= p.Ns) continue;
      const int row = m_tile * BM + r0;
      RowBest rb[2];
      rb[0].begin(p, row, b);
      rb[1].begin(p, row + 8, b);
      for (int nt = nt0; nt < nt1; ++nt) {
        const bool last = nt + 1 == nt1;   // the src chunks may be refilled once this tile's wgmma on them retired
        // one wgmma group stays in flight: the stage of chunk kc - 1 is released once chunk kc has been issued
        int prev = -1;
        for (int kc = 0; kc < wk.k_chunks; ++kc) {
          if (resident && nt == nt0) mbar_wait(a_full_bar(kc), a_phase);
          mbar_wait(full_bar(stage), phase);
          const uint32_t sa = ring_base + stage * lay.stage_bytes;
          const uint32_t a_chunk = resident ? a_base + kc * A_BYTES : sa;
          const uint64_t adesc = wgmma_desc_sw128_kmajor(a_chunk + cg * 64 * 128);
          const uint64_t bdesc = wgmma_desc_sw128_kmajor(sa + b_off);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < BK / UK; ++k)
            wgmma_m64n256k16_f16(d, adesc + 2u * k, bdesc + 2u * k, (kc | k) != 0 ? 1u : 0u);
          wgmma_commit();
          wgmma_wait<1>();
          if (prev >= 0) {
            release(prev);
            if (resident && last) release_a(kc - 1);
          }
          prev = stage;
          if (++stage == stages) { stage = 0; phase ^= 1u; }
        }
        wgmma_wait<0>();
        release(prev);
        if (resident && last) release_a(wk.k_chunks - 1);
        tile_argmax(d, rb, nt * BN, p.Nd, lane);
      }
      rb[0].quad_reduce();
      rb[1].quad_reduce();
      if ((lane & 3) == 0) {
        rb[0].publish(p, row, b);
        rb[1].publish(p, row + 8, b);
      }
      a_phase ^= 1u;
    }
  }
}

int launch(const CUtensorMap& ta, const CUtensorMap& tb, const Items& wk, const Layout& lay, const Args& p, int sms,
           cudaStream_t stream) {
  const size_t smem = lay.smem_bytes();
  // shared-memory opt-in: once per device, at the limit (a per-function, per-device attribute)
  static bool opted[64];
  int dev = 0;
  int rc = cuda_rc(cudaGetDevice(&dev));
  if (rc) return rc;
  if (dev < 0 || dev >= 64 || !opted[dev]) {
    rc = cuda_rc(cudaFuncSetAttribute(sim_argmax_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      static_cast<int>(SMEM_LIMIT)));
    if (rc) return rc;
    if (dev >= 0 && dev < 64) opted[dev] = true;
  }
  const int grid = wk.total < sms ? wk.total : sms;
  sim_argmax_kernel<<<grid, THREADS, smem, stream>>>(ta, tb, wk, lay, p);
  return launch_rc();
}
}  // namespace ka

// ---------------------------------------------------------------------------------------------
// Verification twin on CUDA cores: one thread per src row, dst rows staged through shared memory,
// sequential fp32 FMA over K.  O(Ns*Nd*C) scalar work — for tests only.
__global__ void sim_argmax_simt_kernel(const __half* __restrict__ a, const __half* __restrict__ bm, int B,
                                       int Ns, int Nd, int C, int align_batch, unsigned long long* keys) {
  extern __shared__ __half sb[];  // [TJ][C]
  constexpr int TJ = 32;
  const int b = blockIdx.y;
  const int row = blockIdx.x * blockDim.x + threadIdx.x;
  const __half* arow = a + (static_cast<size_t>(b) * Ns + (row < Ns ? row : 0)) * C;
  float best = -INFINITY;
  uint32_t best_idx = 0xFFFFFFFFu;
  for (int j0 = 0; j0 < Nd; j0 += TJ) {
    const int nj = min(TJ, Nd - j0);
    __syncthreads();
    for (int e = threadIdx.x; e < nj * C; e += blockDim.x)
      sb[e] = bm[(static_cast<size_t>(b) * Nd + j0) * C + e];
    __syncthreads();
    if (row < Ns) {
      for (int j = 0; j < nj; ++j) {
        float acc = 0.f;
        for (int k = 0; k < C; ++k) acc = fmaf(__half2float(arow[k]), __half2float(sb[j * C + k]), acc);
        const float hv = __half2float(__float2half_rn(acc));
        if (hv > best) { best = hv; best_idx = j0 + j; }
      }
    }
  }
  if (row < Ns && best_idx != 0xFFFFFFFFu) {
    const uint32_t hb = static_cast<uint32_t>(__half_as_ushort(__float2half_rn(best)));
    const uint32_t arg = align_batch ? static_cast<uint32_t>(b) * Nd + best_idx : best_idx;
    const size_t o = (align_batch ? 0 : static_cast<size_t>(b) * Ns) + row;
    atomicMax(keys + o, static_cast<unsigned long long>(pack_key(hb, arg)));
  }
}

int check_args(const void* a, const void* b, int B, int Ns, int Nd, int C, const void* keys) {
  if (!a || !b || !keys) return VTM_E_NULL;
  if (B <= 0 || Ns <= 0 || Nd <= 0 || C <= 0 || (C % 8) != 0) return VTM_E_SHAPE;
  if (static_cast<long long>(B) * Nd >= 0xFFFFFFFFll) return VTM_E_SHAPE;
  return VTM_OK;
}

}  // namespace
}  // namespace vtm

namespace vtm {
namespace {
// Ns, Nd: the counts, or with counts_dev (device counts) the capacities the buffers and the grid are sized for
int sim_argmax_impl(const void* a_dev, const void* b_dev, int32_t B, int32_t Ns, int32_t Nd, int32_t C,
                    int32_t align_batch, uint64_t* keys_out_dev, void* stream_,
                    const int32_t* counts_dev = nullptr) {
  int rc = check_args(a_dev, b_dev, B, Ns, Nd, C, keys_out_dev);
  if (rc) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int Bp = align_batch ? 1 : B;
  rc = cuda_rc(cudaMemsetAsync(keys_out_dev, 0, sizeof(uint64_t) * static_cast<size_t>(Bp) * Ns, stream));
  if (rc) return rc;

  CUtensorMap ta, tb;
  rc = make_tmap_3d_f16(&ta, a_dev, C, Ns, B, C, static_cast<uint64_t>(Ns) * C, ka::BK, ka::BM);
  if (rc) return rc;
  rc = make_tmap_3d_f16(&tb, b_dev, C, Nd, B, C, static_cast<uint64_t>(Nd) * C, ka::BK, ka::BN);
  if (rc) return rc;
  int sms = 0;
  rc = cached_sm_count(&sms);
  if (rc) return rc;

  ka::Items wk;
  wk.plan(Ns, Nd, C, B, sms, ka::TARGET_ITEMS_PER_SM);
  ka::Layout lay;
  lay.plan(wk.k_chunks);
  ka::Args p;
  p.keys = reinterpret_cast<unsigned long long*>(keys_out_dev);
  p.Ns = Ns; p.Nd = Nd; p.align_batch = align_batch ? 1 : 0;
  p.ld = Ns; p.counts = counts_dev;
  return ka::launch(ta, tb, wk, lay, p, sms, stream);
}
}  // namespace
}  // namespace vtm

extern "C" int vtm_sim_argmax(const void* a_dev, const void* b_dev, int32_t B, int32_t Ns, int32_t Nd,
                              int32_t C, int32_t align_batch, uint64_t* keys_out_dev, void* stream_) {
  return vtm::sim_argmax_impl(a_dev, b_dev, B, Ns, Nd, C, align_batch, keys_out_dev, stream_);
}

extern "C" int vtm_sim_argmax_dev(const void* a_dev, const void* b_dev, int32_t B, int32_t ns_cap, int32_t nd_cap,
                                  int32_t C, int32_t align_batch, const int32_t* counts_dev, uint64_t* keys_out_dev,
                                  void* stream_) {
  if (!counts_dev) return VTM_E_NULL;
  return vtm::sim_argmax_impl(a_dev, b_dev, B, ns_cap, nd_cap, C, align_batch, keys_out_dev, stream_, counts_dev);
}

extern "C" int vtm_sim_argmax_simt(const void* a_dev, const void* b_dev, int32_t B, int32_t Ns,
                                   int32_t Nd, int32_t C, int32_t align_batch, uint64_t* keys_out_dev,
                                   void* stream_) {
  using namespace vtm;
  int rc = check_args(a_dev, b_dev, B, Ns, Nd, C, keys_out_dev);
  if (rc) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int Bp = align_batch ? 1 : B;
  rc = cuda_rc(cudaMemsetAsync(keys_out_dev, 0, sizeof(uint64_t) * static_cast<size_t>(Bp) * Ns, stream));
  if (rc) return rc;
  const int threads = 128;
  dim3 grid((Ns + threads - 1) / threads, B);
  const size_t smem = static_cast<size_t>(32) * C * sizeof(__half);
  if (smem > 48 * 1024) {
    rc = cuda_rc(cudaFuncSetAttribute(sim_argmax_simt_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      static_cast<int>(smem)));
    if (rc) return rc;
  }
  sim_argmax_simt_kernel<<<grid, threads, smem, stream>>>(
      static_cast<const __half*>(a_dev), static_cast<const __half*>(b_dev), B, Ns, Nd, C,
      align_batch ? 1 : 0, reinterpret_cast<unsigned long long*>(keys_out_dev));
  return launch_rc();
}

extern "C" uint16_t vtm_key_score_half_bits(uint64_t key) {
  return static_cast<uint16_t>(vtm::ordered_to_half_bits(static_cast<uint32_t>(key >> 32)));
}
extern "C" uint32_t vtm_key_arg(uint64_t key) { return 0xFFFFFFFFu - static_cast<uint32_t>(key & 0xFFFFFFFFull); }
