// Persistent warp-specialised wgmma GEMM mainloop for sm_90a, shared by the projection GEMMs of KD (QKV, output,
// GEGLU, residual: fp16 store epilogues).  KA (similarity + row arg-max) has its own kernel in sim_argmax.cu.
//
//   D[b][m, n] = sum_k A[b][m, k] * Bm[b][n, k]        fp16 operands (K-major), fp32 accumulators
//
// One CTA = 384 threads, three warpgroups: warpgroup 0 is the TMA producer (one lane issues), warpgroups 1 and 2 are
// the MMA consumers, each owning 64 rows of the 128 x BN tile (wgmma m64n128k16, accumulators in registers).
// Shared memory: STAGES x (A tile 128x64 + B tile BNx64) fp16, 128-byte swizzled by TMA and read in place by wgmma
// through shared-memory descriptors.  The producer runs ahead across tile and work-item boundaries, so the loads of
// tile i+1 overlap the epilogue of tile i.
// A work item is (m_tile, b, [nt0, nt1)); CTAs stride over work items (persistent grid = #SMs).
//
// K tail (TAIL = true): after its k_chunks chunks of (A, Bm) the producer loads wk.t_chunks further chunks from a second
// operand pair (T [M, R] through tmap_t, U [N, R] through tmap_u) into the same ring, and the consumers add them to the
// same accumulators:  D = [A | T] [Bm | U]^T.  This is how a LoRA's low-rank update x D^T U^T joins its projection
// (T = x D^T, computed beforehand): R extra K columns, every epilogue unchanged.  TMA zero-fills the boxes past R, so the
// stage's byte count is the same as for a main chunk.  TAIL = false compiles to the plain mainloop.
//
// Epilogues read one ROW per thread: after its mainloop a warpgroup writes its fp32 accumulators to a row-major
// staging area in shared memory, and thread t of the warpgroup then owns row (t % 64) and column half (t / 64) of its
// 64 rows, so that a warp holds 32 consecutive rows of one half.
//
// Epilogue policy `Epi` (all members __device__, called by every consumer thread):
//   static constexpr uint32_t SCRATCH_PER_WARP;                      // per-warp shared staging for stores (or 0)
//   static constexpr bool WHOLE_ROWS;                                // true: the threads of column half 0 take all BN
//                                                                    // columns of their row and those of half 1 idle
//   void begin(int m_tile, int b, int row_in_tile);                  // new work item
//   void tile(const gemm::Acc& acc, int col0, int ncols);           // this thread's row of a finished accumulator:
//                                                                    // acc.ld64(cb, r) gives columns [cb, cb + 64) of
//                                                                    // the slice, col0 = global n of its first column
//   void end(int m_tile, int b, int row_in_tile);                    // work item finished
#pragma once
#include "common.cuh"
#include "ptx.cuh"

namespace vtm {
namespace gemm {

constexpr int BM = 128;
constexpr int BN = 128;
constexpr int BK = 64;
constexpr int UK = 16;
constexpr int CONSUMER_WARPS = 8;
constexpr int THREADS = 384;
constexpr uint32_t A_BYTES = BM * BK * 2;
constexpr uint32_t B_BYTES = BN * BK * 2;
constexpr uint32_t STAGE_BYTES = A_BYTES + B_BYTES;
// fp32 staging row pitch: BN + 4 floats keeps the 16-byte row reads of eight consecutive rows on distinct banks
constexpr int ACC_PITCH = BN + 4;
constexpr uint32_t ACC_BYTES = BM * ACC_PITCH * 4;
constexpr size_t SMEM_LIMIT = 227 * 1024;   // opt-in shared memory per block on sm_90

template <uint32_t SCRATCH_PER_WARP>
struct Cfg {
  static constexpr size_t FIXED = 1024 + ACC_BYTES + CONSUMER_WARPS * SCRATCH_PER_WARP + 256;
  static constexpr int STAGES_FIT = static_cast<int>((SMEM_LIMIT - FIXED) / STAGE_BYTES);
  static constexpr int STAGES = STAGES_FIT > 6 ? 6 : STAGES_FIT;
  static_assert(STAGES >= 2, "shared memory too small for a two-stage ring");
  static constexpr size_t SMEM_BYTES = FIXED + static_cast<size_t>(STAGES) * STAGE_BYTES;
};

// This thread's row of the staged accumulator tile, starting at the first column of its slice.
struct Acc {
  uint32_t row_addr;
  __device__ __forceinline__ void ld64(int cb, uint32_t (&r)[64]) const {
#pragma unroll
    for (int q = 0; q < 16; ++q)
      asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
                   : "=r"(r[4 * q]), "=r"(r[4 * q + 1]), "=r"(r[4 * q + 2]), "=r"(r[4 * q + 3])
                   : "r"(row_addr + static_cast<uint32_t>(cb + 4 * q) * 4u)
                   : "memory");
  }
};

struct Work {
  int batches;          // B
  int m_tiles, n_tiles;
  int tiles_per_split, n_splits;
  int k_chunks;
  int t_chunks;         // K-tail chunks (TAIL kernels only): ceil(R / BK)
  int total;
  // Order of the work items.  0: m tile fastest.  1: n split fastest (plain GEMMs): the splits of one m tile run on
  // neighbouring CTAs at the same time, so the A tile comes from HBM once and from L2 afterwards.
  int n_fastest;
  __host__ void plan(int M, int N, int K, int B, int sms, int target_items_per_sm, int min_tiles) {
    batches = B;
    n_fastest = 0;
    m_tiles = (M + BM - 1) / BM;
    n_tiles = (N + BN - 1) / BN;
    k_chunks = (K + BK - 1) / BK;
    t_chunks = 0;
    const long long base = static_cast<long long>(m_tiles) * B;
    int s = 1;
    while (base * s < static_cast<long long>(target_items_per_sm) * sms && s * 2 <= n_tiles &&
           n_tiles / (s * 2) >= min_tiles)
      s *= 2;
    tiles_per_split = (n_tiles + s - 1) / s;
    n_splits = (n_tiles + tiles_per_split - 1) / tiles_per_split;
    total = static_cast<int>(base * n_splits);
  }
  __device__ __forceinline__ void decode(int w, int* m_tile, int* b, int* nt0, int* nt1) const {
    int sp;
    if (n_fastest) {
      sp = w % n_splits;
      const int rest = w / n_splits;
      *m_tile = rest % m_tiles;
      *b = rest / m_tiles;
    } else {
      *m_tile = w % m_tiles;
      const int rest = w / m_tiles;
      *b = rest % batches;
      sp = rest / batches;
    }
    *nt0 = sp * tiles_per_split;
    const int e = *nt0 + tiles_per_split;
    *nt1 = e < n_tiles ? e : n_tiles;
  }
};


// ---------------------------------------------------------------------------------------------------------
// Row-contiguous stores for epilogues that write the tile to global memory.  A thread holds ONE row of the tile, so a
// direct 16-byte store per thread would touch 32 different cache lines per instruction.  The warp's 32 rows x 64 fp16
// columns go through a 4 KB XOR-swizzled staging area instead: each thread writes its row as eight 16-byte chunks
// (chunk k at slot k ^ (row & 7): conflict-free), then lane l reads chunk l & 7 of row 4 i + l / 8, so that eight
// consecutive lanes store 128 contiguous bytes of one row.
constexpr uint32_t STAGE_STORE_BYTES = 32 * 128;
template <class F>
__device__ __forceinline__ void warp_store_rows64(uint32_t scratch, const uint32_t (&pk)[32], F&& store) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int k = 0; k < 8; ++k)
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(scratch + lane * 128 + ((k ^ (lane & 7)) << 4)),
                 "r"(pk[4 * k]), "r"(pk[4 * k + 1]), "r"(pk[4 * k + 2]), "r"(pk[4 * k + 3])
                 : "memory");
  __syncwarp();
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int r = 4 * i + (lane >> 3), kk = lane & 7;
    uint4 v;
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "r"(scratch + r * 128 + ((kk ^ (r & 7)) << 4))
                 : "memory");
    store(r, kk * 8, v);   // row within the warp's 32, first of 8 columns within the 64
  }
  __syncwarp();
}

// The K tail's tensor maps as one kernel parameter: empty without a tail, so that the plain kernels take the same
// parameters as before the tail existed.
template <bool TAIL>
struct TailMaps {
  CUtensorMap t, u;
};
template <>
struct TailMaps<false> {};

template <class Epi, bool TAIL>
__global__ void __launch_bounds__(THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
            const __grid_constant__ TailMaps<TAIL> tail, const Work wk, Epi epi) {
  using C = Cfg<Epi::SCRATCH_PER_WARP>;
  constexpr int STAGES = C::STAGES;
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment: required by the 128-byte swizzle pattern shared by TMA and wgmma descriptors
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t acc_base = smem_base + STAGES * STAGE_BYTES;
  const uint32_t scratch_base = acc_base + ACC_BYTES;
  const uint32_t bar_base = scratch_base + CONSUMER_WARPS * Epi::SCRATCH_PER_WARP;
  // 8-byte slots: full[STAGES] | empty[STAGES]
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const int w_first = static_cast<int>(blockIdx.x);
  const int w_step = static_cast<int>(gridDim.x);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    if constexpr (TAIL) {
      tma_prefetch_desc(&tail.t);
      tma_prefetch_desc(&tail.u);
    }
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), CONSUMER_WARPS);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int w = w_first; w < wk.total; w += w_step) {
        int m_tile, b, nt0, nt1;
        wk.decode(w, &m_tile, &b, &nt0, &nt1);
        for (int nt = nt0; nt < nt1; ++nt) {
          const int kn = TAIL ? wk.k_chunks + wk.t_chunks : wk.k_chunks;
          for (int kc = 0; kc < kn; ++kc) {
            const uint32_t sa = smem_base + stage * STAGE_BYTES;
            mbar_wait(empty_bar(stage), phase ^ 1u);
            mbar_arrive_expect_tx(full_bar(stage), STAGE_BYTES);
            if constexpr (TAIL) {
              if (kc < wk.k_chunks) {
                tma_load_3d(sa, &tmap_a, full_bar(stage), kc * BK, m_tile * BM, b);
                tma_load_3d(sa + A_BYTES, &tmap_b, full_bar(stage), kc * BK, nt * BN, b);
              } else {
                const int kt = kc - wk.k_chunks;
                tma_load_3d(sa, &tail.t, full_bar(stage), kt * BK, m_tile * BM, b);
                tma_load_3d(sa + A_BYTES, &tail.u, full_bar(stage), kt * BK, nt * BN, b);
              }
            } else {
              tma_load_3d(sa, &tmap_a, full_bar(stage), kc * BK, m_tile * BM, b);
              tma_load_3d(sa + A_BYTES, &tmap_b, full_bar(stage), kc * BK, nt * BN, b);
            }
            if (++stage == STAGES) { stage = 0; phase ^= 1u; }
          }
        }
      }
    }
  } else {
    // ===================== MMA + epilogue =====================
    setmaxnreg_inc<232>();
    const int cg = wg - 1;                        // which 64 rows of the tile
    const int t = threadIdx.x - 128 * wg;         // thread within the warpgroup
    const int wq = t >> 5;                        // warp within the warpgroup
    const int row_in_tile = cg * 64 + (t & 63);
    const int half = t >> 6;
    const bool active = !Epi::WHOLE_ROWS || half == 0;
    const int slice_cols = Epi::WHOLE_ROWS ? BN : BN / 2;
    const int slice_col0 = Epi::WHOLE_ROWS ? 0 : half * (BN / 2);
    const Acc acc{acc_base + static_cast<uint32_t>(row_in_tile * ACC_PITCH + slice_col0) * 4u};
    Epi e = epi;  // per-thread mutable copy of the policy (kernel parameters are read-only)
    if constexpr (Epi::SCRATCH_PER_WARP > 0)
      e.set_scratch(scratch_base + static_cast<uint32_t>(warp - 4) * Epi::SCRATCH_PER_WARP);
    int stage = 0;
    uint32_t phase = 0;
    float d[64];
    // smem slot reusable: this warp's MMAs reading it have retired
    auto release = [&](int st) {
      __syncwarp();
      if (lane == 0) mbar_arrive(empty_bar(st));
    };
    for (int w = w_first; w < wk.total; w += w_step) {
      int m_tile, b, nt0, nt1;
      wk.decode(w, &m_tile, &b, &nt0, &nt1);
      e.begin(m_tile, b, row_in_tile);
      for (int nt = nt0; nt < nt1; ++nt) {
        // one wgmma group stays in flight: the stage of chunk kc - 1 is released once chunk kc has been issued
        int prev = -1;
        const int kn = TAIL ? wk.k_chunks + wk.t_chunks : wk.k_chunks;
        for (int kc = 0; kc < kn; ++kc) {
          mbar_wait(full_bar(stage), phase);
          const uint32_t sa = smem_base + stage * STAGE_BYTES;
          const uint64_t adesc = wgmma_desc_sw128_kmajor(sa + cg * 64 * 128);
          const uint64_t bdesc = wgmma_desc_sw128_kmajor(sa + A_BYTES);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < BK / UK; ++k)
            wgmma_m64n128k16_f16(d, adesc + 2u * k, bdesc + 2u * k, (kc | k) != 0 ? 1u : 0u);
          wgmma_commit();
          wgmma_wait<1>();
          if (prev >= 0) release(prev);
          prev = stage;
          if (++stage == STAGES) { stage = 0; phase ^= 1u; }
        }
        wgmma_wait<0>();
        release(prev);
        // stage the accumulators row-major (the previous tile's epilogue of this warpgroup must be done reading)
        bar_sync_named(1 + cg, 128);
        {
          const int r0 = cg * 64 + wq * 16 + (lane >> 2);
          const uint32_t base = acc_base + static_cast<uint32_t>(r0 * ACC_PITCH + 2 * (lane & 3)) * 4u;
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(base + 32u * j), "f"(d[4 * j]), "f"(d[4 * j + 1])
                         : "memory");
            asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(base + 8u * ACC_PITCH * 4u + 32u * j),
                         "f"(d[4 * j + 2]), "f"(d[4 * j + 3])
                         : "memory");
          }
        }
        bar_sync_named(1 + cg, 128);
        if (active) e.tile(acc, nt * BN + slice_col0, slice_cols);
      }
      e.end(m_tile, b, row_in_tile);
    }
  }
}

template <class Epi, bool TAIL>
inline int launch_impl(const CUtensorMap& ta, const CUtensorMap& tb, const TailMaps<TAIL>& tail, const Work& wk,
                       const Epi& epi, int sms, cudaStream_t stream) {
  using C = Cfg<Epi::SCRATCH_PER_WARP>;
  const size_t smem = C::SMEM_BYTES;
  // shared-memory opt-in: once per instantiation and device (a per-function, per-device attribute; immutable afterwards)
  static bool opted[64];
  int dev = 0;
  int rc = cuda_rc(cudaGetDevice(&dev));
  if (rc) return rc;
  if (dev < 0 || dev >= 64 || !opted[dev]) {
    rc = cuda_rc(cudaFuncSetAttribute(gemm_kernel<Epi, TAIL>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      static_cast<int>(smem)));
    if (rc) return rc;
    if (dev >= 0 && dev < 64) opted[dev] = true;
  }
  const int grid = wk.total < sms ? wk.total : sms;
  gemm_kernel<Epi, TAIL><<<grid, THREADS, smem, stream>>>(ta, tb, tail, wk, epi);
  return launch_rc();
}

template <class Epi>
inline int launch(const CUtensorMap& ta, const CUtensorMap& tb, const Work& wk, const Epi& epi, int sms,
                  cudaStream_t stream) {
  return launch_impl<Epi, false>(ta, tb, TailMaps<false>{}, wk, epi, sms, stream);
}

// With the K tail: tt / tu from make_tail.
template <class Epi>
inline int launch_tail(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tt, const CUtensorMap& tu,
                       const Work& wk, const Epi& epi, int sms, cudaStream_t stream) {
  return launch_impl<Epi, true>(ta, tb, TailMaps<true>{tt, tu}, wk, epi, sms, stream);
}

// The K tail of a GEMM with M rows and N columns: T [M, R] and U [N, R] fp16 (R % 8 == 0, 16-byte aligned), and the
// tail's chunk count in wk (after wk.plan).
inline int make_tail(const void* t_dev, const void* u_dev, int R, int M, int N, CUtensorMap* tt, CUtensorMap* tu,
                     Work* wk) {
  int rc = make_tmap_3d_f16(tt, t_dev, R, M, 1, R, static_cast<uint64_t>(M) * R, BK, BM);
  if (rc) return rc;
  rc = make_tmap_3d_f16(tu, u_dev, R, N, 1, R, static_cast<uint64_t>(N) * R, BK, BN);
  if (rc) return rc;
  wk->t_chunks = (R + BK - 1) / BK;
  return 0;
}

inline int device_sms(int* sms) { return cached_sm_count(sms); }

}  // namespace gemm
}  // namespace vtm
