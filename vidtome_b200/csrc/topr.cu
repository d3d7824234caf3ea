// KB — top-r selection and index-map composition.
//
// KB1: stable descending sort of the Ns row maxima of each sample (vidtome/merge.py:98,113,402,417
// `node_max.argsort(dim=-1, descending=True)`; stable = ties keep ascending src-row order).  The sort
// key is the 16-bit order-preserving image of the fp16 maximum already stored in bits 32..47 of the
// KA key, so two LSD radix passes of 8 bits suffice.  Each pass is: per-tile digit histogram ->
// exclusive scan over (digit descending, tile ascending) -> stable scatter.  A tile is 1024 elements
// handled by 1024 threads (one element per thread, thread order = element order), ranks inside a tile
// come from __match_any_sync within a warp plus a per-digit prefix over the 32 warps.
//
// KB2: one pass over max(N0, N_next) entries that applies the level's match to the composed maps
// (see include/vidtome_b200.h).  Decode: expands the match into the reference's int64 index tensors.
#include "common.cuh"
#include "ptx.cuh"

namespace vtm {
namespace {

constexpr int TILE = 1024;
constexpr int NW = TILE / 32;

__device__ __forceinline__ int digit_of(uint32_t key16, int pass) {
  // descending order: larger key first -> bucket index = 255 - digit
  return 255 - static_cast<int>((key16 >> (8 * pass)) & 0xFFu);
}

// Rank of each thread's element among the tile's elements with the same bucket and a lower thread
// index; also the tile's bucket counts (in s_tot[256]).  Must be called by all 1024 threads.
__device__ __forceinline__ int tile_rank(int bucket, bool valid, uint32_t (*s_cnt)[256], uint32_t* s_tot) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < NW * 256; i += TILE) (&s_cnt[0][0])[i] = 0;
  __syncthreads();
  // invalid (padding) threads use a bucket id outside 0..255 so that they match only each other
  const int mb = valid ? bucket : 256;
  const uint32_t peers = __match_any_sync(0xffffffffu, mb);
  const int in_warp = __popc(peers & ((1u << lane) - 1u));
  if (valid && in_warp == 0) s_cnt[warp][bucket] = __popc(peers);
  __syncthreads();
  if (threadIdx.x < 256) {
    uint32_t run = 0;
#pragma unroll 4
    for (int w = 0; w < NW; ++w) {
      const uint32_t c = s_cnt[w][threadIdx.x];
      s_cnt[w][threadIdx.x] = run;
      run += c;
    }
    s_tot[threadIdx.x] = run;
  }
  __syncthreads();
  return valid ? static_cast<int>(s_cnt[warp][bucket]) + in_warp : 0;
}

// pass 0 reads the KA keys (element id = src row); pass 1 reads the (key16, id) pairs of pass 0.
template <int PASS>
__global__ void __launch_bounds__(TILE)
radix_hist_kernel(const unsigned long long* __restrict__ keys, const uint16_t* __restrict__ k_in, int Ns,
                  int tiles, uint32_t* __restrict__ hist /* [Bp][256][tiles] */, int ld, const int* __restrict__ ns_dev) {
  __shared__ uint32_t s_cnt[NW][256];
  __shared__ uint32_t s_tot[256];
  if (ns_dev) Ns = __ldg(ns_dev);
  const int b = blockIdx.y, tile = blockIdx.x;
  const int e = tile * TILE + threadIdx.x;
  const bool valid = e < Ns;
  uint32_t k16 = 0;
  if (valid)
    k16 = PASS == 0 ? static_cast<uint32_t>(keys[static_cast<size_t>(b) * ld + e] >> 32) & 0xFFFFu
                    : k_in[static_cast<size_t>(b) * ld + e];
  tile_rank(digit_of(k16, PASS), valid, s_cnt, s_tot);
  if (threadIdx.x < 256)
    hist[(static_cast<size_t>(b) * 256 + threadIdx.x) * tiles + tile] = s_tot[threadIdx.x];
}

// exclusive scan of hist[b][bucket][tile] in (bucket, tile) order; one CTA per sample.
__global__ void __launch_bounds__(1024) radix_scan_kernel(uint32_t* __restrict__ hist, int tiles) {
  __shared__ uint32_t s_part[1024];
  const int b = blockIdx.x;
  const int n = 256 * tiles;
  uint32_t* h = hist + static_cast<size_t>(b) * n;
  const int per = (n + 1023) / 1024;
  const int lo = threadIdx.x * per, hi = min(lo + per, n);
  uint32_t sum = 0;
  for (int i = lo; i < hi; ++i) sum += h[i];
  s_part[threadIdx.x] = sum;
  __syncthreads();
  // Hillis-Steele inclusive scan over 1024 partials
  for (int off = 1; off < 1024; off <<= 1) {
    uint32_t v = threadIdx.x >= off ? s_part[threadIdx.x - off] : 0;
    __syncthreads();
    s_part[threadIdx.x] += v;
    __syncthreads();
  }
  uint32_t run = s_part[threadIdx.x] - sum;
  for (int i = lo; i < hi; ++i) {
    const uint32_t c = h[i];
    h[i] = run;
    run += c;
  }
}

template <int PASS>
__global__ void __launch_bounds__(TILE)
radix_scatter_kernel(const unsigned long long* __restrict__ keys, const uint16_t* __restrict__ k_in,
                     const int* __restrict__ id_in, int Ns, int tiles, const uint32_t* __restrict__ base,
                     uint16_t* __restrict__ k_out, int* __restrict__ id_out, int* __restrict__ rank_out, int ld,
                     const int* __restrict__ ns_dev) {
  __shared__ uint32_t s_cnt[NW][256];
  __shared__ uint32_t s_tot[256];
  if (ns_dev) Ns = __ldg(ns_dev);
  const int b = blockIdx.y, tile = blockIdx.x;
  const int e = tile * TILE + threadIdx.x;
  const bool valid = e < Ns;
  uint32_t k16 = 0;
  int id = e;
  if (valid) {
    if (PASS == 0) {
      k16 = static_cast<uint32_t>(keys[static_cast<size_t>(b) * ld + e] >> 32) & 0xFFFFu;
    } else {
      k16 = k_in[static_cast<size_t>(b) * ld + e];
      id = id_in[static_cast<size_t>(b) * ld + e];
    }
  }
  const int bucket = digit_of(k16, PASS);
  const int r = tile_rank(bucket, valid, s_cnt, s_tot);
  if (valid) {
    const uint32_t pos = base[(static_cast<size_t>(b) * 256 + bucket) * tiles + tile] + r;
    const size_t o = static_cast<size_t>(b) * ld + pos;
    if (PASS == 0) {
      k_out[o] = static_cast<uint16_t>(k16);
      id_out[o] = id;
    } else {
      id_out[o] = id;                                         // edge[pos] = src row
      rank_out[static_cast<size_t>(b) * ld + id] = static_cast<int>(pos);  // rank[src row] = pos
    }
  }
}

// ---------------------------------------------------------------- KB2 compose
__global__ void __launch_bounds__(256)
compose_maps_kernel(Split sp, int r, int Bp, const unsigned long long* __restrict__ keys,
                    const int* __restrict__ edge, const int* __restrict__ rank, const int* __restrict__ mu_in,
                    const int* __restrict__ pi_in, int pi_offset, int N0, int* __restrict__ mu_out,
                    int* __restrict__ pi_out, const int* __restrict__ counts = nullptr) {
  // device counts (mode 2): keys / edge / rank have row stride cap, mu_out row stride src_len + gcap
  const int ldk = sp.cap ? sp.cap : sp.Ns;
  const int ldmu = sp.cap ? sp.src_len + sp.gcap : (sp.Ns - r) + sp.Nd;
  resolve_split<true>(sp);
  if (counts) r = __ldg(counts + 2);
  const int b = blockIdx.y;
  const int Ns = sp.Ns, Nd = sp.Nd;
  const int unm = Ns - r;
  const int Lnext = unm + Nd;
  const unsigned long long* kb = keys + static_cast<size_t>(b) * ldk;
  const int* eb = edge + static_cast<size_t>(b) * ldk;
  const int* rb = rank + static_cast<size_t>(b) * ldk;
  const int* mub = mu_in ? mu_in + static_cast<size_t>(b) * sp.N : nullptr;
  const int* pib = pi_in ? pi_in + static_cast<size_t>(b) * N0 : nullptr;
  const int n_iter = Lnext > N0 ? Lnext : N0;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n_iter; t += gridDim.x * blockDim.x) {
    if (t < Lnext) {
      // merged sequence = [unmerged src in edge order | dst]  (merge.py:124,133)
      const int pos = t < unm ? src_pos<true>(sp, eb[r + t]) : dst_pos<true>(sp, t - unm);
      mu_out[static_cast<size_t>(b) * ldmu + t] = mub ? mub[pos] : pos;
    }
    if (t < N0 && (pib || t < sp.N)) {             // without pi_in, positions past the sequence have no image
      const int p = (pib ? pib[t] : t) + pi_offset;  // position in this level's sequence
      int idx;
      int np;
      if (pos_to_part<true>(sp, p, &idx)) {
        np = unm + idx;                                // dst j -> merged[unm + j]      (merge.py:146)
      } else {
        const int k = rb[idx];
        if (k < r) {                                   // merged away: takes its dst's value (merge.py:143,153)
          const uint32_t arg = 0xFFFFFFFFu - static_cast<uint32_t>(kb[idx] & 0xFFFFFFFFull);
          np = unm + static_cast<int>(arg % static_cast<uint32_t>(Nd));
        } else {
          np = k - r;                                  // kept: merged[k - r]          (merge.py:149)
        }
      }
      pi_out[static_cast<size_t>(b) * N0 + t] = np;
    }
  }
}

__global__ void __launch_bounds__(256)
decode_match_kernel(const unsigned long long* __restrict__ keys, const int* __restrict__ edge, int Ns, int Nd,
                    int r, long long* __restrict__ unm_idx, long long* __restrict__ src_idx,
                    long long* __restrict__ dst_idx, uint16_t* __restrict__ node_max,
                    long long* __restrict__ node_idx) {
  const int b = blockIdx.y;
  const unsigned long long* kb = keys + static_cast<size_t>(b) * Ns;
  const int* eb = edge + static_cast<size_t>(b) * Ns;
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < Ns; k += gridDim.x * blockDim.x) {
    const int i = eb[k];
    const uint32_t arg = 0xFFFFFFFFu - static_cast<uint32_t>(kb[i] & 0xFFFFFFFFull);
    if (k < r) {
      if (src_idx) src_idx[static_cast<size_t>(b) * r + k] = i;
      if (dst_idx) dst_idx[static_cast<size_t>(b) * r + k] = arg % static_cast<uint32_t>(Nd);
    } else if (unm_idx) {
      unm_idx[static_cast<size_t>(b) * (Ns - r) + (k - r)] = i;
    }
    // node_max / node_idx are indexed by src row, not by rank
    const unsigned long long kk = kb[k];
    if (node_max) node_max[static_cast<size_t>(b) * Ns + k] =
        static_cast<uint16_t>(ordered_to_half_bits(static_cast<uint32_t>(kk >> 32)));
    if (node_idx) node_idx[static_cast<size_t>(b) * Ns + k] =
        0xFFFFFFFFu - static_cast<uint32_t>(kk & 0xFFFFFFFFull);
  }
}

// ---------------------------------------------------------------- fused single-launch sort
// Same algorithm in ONE cooperative launch: every CTA keeps its 1024-element tile for both passes, the
// per-(digit, tile) histogram table is exchanged through global memory and each CTA scans the part of it it
// needs; phases are separated by a grid-wide barrier (monotonic counter, co-residency guaranteed by
// cudaLaunchCooperativeKernel).  Used when tiles * Bp CTAs fit on the device at once.
__device__ __forceinline__ void grid_barrier(unsigned int* ctr, unsigned int target) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(ctr, 1u);
    unsigned int v;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory");
    } while (v < target);
    __threadfence();
  }
  __syncthreads();
}

// exclusive prefix of hist[bucket][tile] in (bucket, tile) order for ONE (bucket, tile) pair per thread:
// thread t (t < 256) gets the base of bucket t for this CTA's tile.  All 1024 threads share the column sums: thread
// (bucket = t % 256, quarter = t / 256) adds a quarter of the tiles with independent loads in flight (the first version
// walked all tiles from one thread per bucket: a chain of ~50 dependent L2 latencies per pass, the bulk of the kernel).
__device__ __forceinline__ uint32_t bucket_base(const uint32_t* __restrict__ h /* [256][tiles] */, int tiles,
                                                int my_tile, uint32_t* s_scan /* [256] */, uint32_t (*s_part)[256] /* [8][256] */) {
  {
    const int bucket = threadIdx.x & 255, quarter = threadIdx.x >> 8;
    const int t0 = quarter * tiles / 4, t1 = (quarter + 1) * tiles / 4;
    const uint32_t* row = h + static_cast<size_t>(bucket) * tiles;
    uint32_t tot = 0, bef = 0;
#pragma unroll 4
    for (int t = t0; t < t1; ++t) {
      const uint32_t c = __ldcg(row + t);
      tot += c;
      bef += t < my_tile ? c : 0u;
    }
    s_part[quarter][bucket] = tot;
    s_part[4 + quarter][bucket] = bef;
  }
  __syncthreads();
  uint32_t total = 0, before = 0;
  if (threadIdx.x < 256) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      total += s_part[q][threadIdx.x];
      before += s_part[4 + q][threadIdx.x];
    }
    s_scan[threadIdx.x] = total;
  }
  __syncthreads();
  // inclusive scan over the 256 bucket totals (8 warps of 32)
  uint32_t incl = 0;
  if (threadIdx.x < 256) {
    incl = total;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
      if ((threadIdx.x & 31) >= o) incl += v;
    }
  }
  __syncthreads();
  if (threadIdx.x < 256 && (threadIdx.x & 31) == 31) s_scan[threadIdx.x >> 5] = incl;   // warp totals
  __syncthreads();
  uint32_t base = 0;
  if (threadIdx.x < 256) {
    uint32_t warp_off = 0;
    for (int w = 0; w < (threadIdx.x >> 5); ++w) warp_off += s_scan[w];
    base = warp_off + incl - total + before;
  }
  __syncthreads();
  return base;
}

__global__ void __launch_bounds__(TILE)
radix_sort_fused_kernel(const unsigned long long* __restrict__ keys, int Ns, int tiles, uint32_t* hist0,
                        uint32_t* hist1, uint16_t* k_tmp, int* id_tmp, int* __restrict__ edge,
                        int* __restrict__ rank_out, unsigned int* barrier_ctr, int ld, const int* __restrict__ ns_dev) {
  __shared__ uint32_t s_cnt[NW][256];
  __shared__ uint32_t s_tot[256];
  __shared__ uint32_t s_base[256];
  __shared__ uint32_t s_scan[256];
  __shared__ uint32_t s_part[8][256];
  const int b = blockIdx.y, tile = blockIdx.x;
  const unsigned int nblk = gridDim.x * gridDim.y;
  if (ns_dev) Ns = __ldg(ns_dev);
  const size_t row0 = static_cast<size_t>(b) * ld;
  const int e = tile * TILE + threadIdx.x;
  const bool valid = e < Ns;
  // ---- pass 0 (low byte)
  uint32_t k16 = valid ? static_cast<uint32_t>(keys[row0 + e] >> 32) & 0xFFFFu : 0u;
  int bucket = digit_of(k16, 0);
  int r = tile_rank(bucket, valid, s_cnt, s_tot);
  uint32_t* h0 = hist0 + static_cast<size_t>(b) * 256 * tiles;
  if (threadIdx.x < 256) h0[static_cast<size_t>(threadIdx.x) * tiles + tile] = s_tot[threadIdx.x];
  grid_barrier(barrier_ctr, nblk);
  uint32_t base = bucket_base(h0, tiles, tile, s_scan, s_part);
  if (threadIdx.x < 256) s_base[threadIdx.x] = base;
  __syncthreads();
  if (valid) {
    const uint32_t pos = s_base[bucket] + r;
    k_tmp[row0 + pos] = static_cast<uint16_t>(k16);
    id_tmp[row0 + pos] = e;
  }
  grid_barrier(barrier_ctr, 2 * nblk);
  // ---- pass 1 (high byte) on the pass-0 order
  int id = e;
  if (valid) {
    k16 = __ldcg(k_tmp + row0 + e);
    id = __ldcg(id_tmp + row0 + e);
  }
  bucket = digit_of(k16, 1);
  r = tile_rank(bucket, valid, s_cnt, s_tot);
  uint32_t* h1 = hist1 + static_cast<size_t>(b) * 256 * tiles;
  if (threadIdx.x < 256) h1[static_cast<size_t>(threadIdx.x) * tiles + tile] = s_tot[threadIdx.x];
  grid_barrier(barrier_ctr, 3 * nblk);
  base = bucket_base(h1, tiles, tile, s_scan, s_part);
  if (threadIdx.x < 256) s_base[threadIdx.x] = base;
  __syncthreads();
  if (valid) {
    const uint32_t pos = s_base[bucket] + r;
    edge[row0 + pos] = id;
    rank_out[row0 + id] = static_cast<int>(pos);
  }
}

struct SortWs {
  uint32_t* hist;
  uint32_t* hist1;
  uint16_t* k_tmp;
  int* id_tmp;
  unsigned int* barrier;
};
size_t align256(size_t v) { return (v + 255) & ~static_cast<size_t>(255); }
size_t sort_ws_layout(int Bp, int Ns, void* base, SortWs* ws) {
  const int tiles = (Ns + TILE - 1) / TILE;
  size_t off = 0;
  uint8_t* p = static_cast<uint8_t*>(base);
  if (ws) ws->hist = reinterpret_cast<uint32_t*>(p + off);
  off += align256(sizeof(uint32_t) * static_cast<size_t>(Bp) * 256 * tiles);
  if (ws) ws->hist1 = reinterpret_cast<uint32_t*>(p + off);
  off += align256(sizeof(uint32_t) * static_cast<size_t>(Bp) * 256 * tiles);
  if (ws) ws->barrier = reinterpret_cast<unsigned int*>(p + off);
  off += 256;
  if (ws) ws->k_tmp = reinterpret_cast<uint16_t*>(p + off);
  off += align256(sizeof(uint16_t) * static_cast<size_t>(Bp) * Ns);
  if (ws) ws->id_tmp = reinterpret_cast<int*>(p + off);
  off += align256(sizeof(int) * static_cast<size_t>(Bp) * Ns);
  return off;
}

}  // namespace
}  // namespace vtm

extern "C" size_t vtm_topr_workspace_bytes(int32_t Bp, int32_t Ns) {
  if (Bp <= 0 || Ns <= 0) return 0;
  return vtm::sort_ws_layout(Bp, Ns, nullptr, nullptr);
}

namespace vtm {
namespace {
// Ns: the count (ns_dev == NULL) or the capacity and row stride (ns_dev: the count on the device, <= Ns)
int topr_sort_impl(const uint64_t* keys_dev, int32_t Bp, int32_t Ns, const int32_t* ns_dev, int32_t* edge_dev,
                   int32_t* rank_dev, void* ws_dev, size_t ws_bytes, void* stream_) {
  if (!keys_dev || !edge_dev || !rank_dev || !ws_dev) return VTM_E_NULL;
  if (Bp <= 0 || Ns <= 0) return VTM_E_SHAPE;
  SortWs ws;
  if (sort_ws_layout(Bp, Ns, ws_dev, &ws) > ws_bytes) return VTM_E_WS;
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  const int tiles = (Ns + TILE - 1) / TILE;
  const unsigned long long* keys = reinterpret_cast<const unsigned long long*>(keys_dev);
  dim3 grid(tiles, Bp);
  // single cooperative launch when every CTA can be resident at once
  {
    // device facts: looked up once per device ordinal (immutable afterwards)
    static int t_sms[64], t_per_sm[64], t_coop[64];
    int dev = 0, sms = 0, per_sm = 0, coop = 0;
    int rc = cuda_rc(cudaGetDevice(&dev));
    if (rc) return rc;
    if (dev >= 0 && dev < 64 && t_sms[dev] > 0) {
      sms = t_sms[dev]; per_sm = t_per_sm[dev]; coop = t_coop[dev];
    } else {
      cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
      cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev);
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, radix_sort_fused_kernel, TILE, 0);
      if (dev >= 0 && dev < 64 && sms > 0) { t_per_sm[dev] = per_sm; t_coop[dev] = coop; t_sms[dev] = sms; }
    }
    if (coop && static_cast<long long>(tiles) * Bp <= static_cast<long long>(sms) * per_sm) {
      rc = cuda_rc(cudaMemsetAsync(ws.barrier, 0, sizeof(unsigned int), st));
      if (rc) return rc;
      int ns = Ns, tl = tiles;
      // A plain launch: every CTA of the grid fits on the device at once (checked above), and kernels ahead of this one
      // — earlier in the stream, or on other streams — finish without depending on it, so all CTAs become resident
      // and the spin barriers cannot deadlock.  The cooperative launch API adds host-side validation per call and a
      // heavier launch path; measured r02.
      (void)ns; (void)tl;
      radix_sort_fused_kernel<<<grid, TILE, 0, st>>>(keys, Ns, tiles, ws.hist, ws.hist1, ws.k_tmp, ws.id_tmp, edge_dev,
                                                    rank_dev, ws.barrier, Ns, ns_dev);
      return launch_rc();
    }
  }
  radix_hist_kernel<0><<<grid, TILE, 0, st>>>(keys, nullptr, Ns, tiles, ws.hist, Ns, ns_dev);
  radix_scan_kernel<<<Bp, 1024, 0, st>>>(ws.hist, tiles);
  radix_scatter_kernel<0><<<grid, TILE, 0, st>>>(keys, nullptr, nullptr, Ns, tiles, ws.hist, ws.k_tmp,
                                                 ws.id_tmp, nullptr, Ns, ns_dev);
  radix_hist_kernel<1><<<grid, TILE, 0, st>>>(nullptr, ws.k_tmp, Ns, tiles, ws.hist, Ns, ns_dev);
  radix_scan_kernel<<<Bp, 1024, 0, st>>>(ws.hist, tiles);
  radix_scatter_kernel<1><<<grid, TILE, 0, st>>>(nullptr, ws.k_tmp, ws.id_tmp, Ns, tiles, ws.hist, nullptr,
                                                 edge_dev, rank_dev, Ns, ns_dev);
  return launch_rc();
}
}  // namespace
}  // namespace vtm

extern "C" int vtm_topr_sort(const uint64_t* keys_dev, int32_t Bp, int32_t Ns, int32_t* edge_dev,
                             int32_t* rank_dev, void* ws_dev, size_t ws_bytes, void* stream_) {
  return vtm::topr_sort_impl(keys_dev, Bp, Ns, nullptr, edge_dev, rank_dev, ws_dev, ws_bytes, stream_);
}

extern "C" int vtm_topr_sort_dev(const uint64_t* keys_dev, int32_t Bp, int32_t ns_cap, const int32_t* counts_dev,
                                 int32_t* edge_dev, int32_t* rank_dev, void* ws_dev, size_t ws_bytes, void* stream_) {
  if (!counts_dev) return VTM_E_NULL;
  return vtm::topr_sort_impl(keys_dev, Bp, ns_cap, counts_dev, edge_dev, rank_dev, ws_dev, ws_bytes, stream_);
}

extern "C" int vtm_compose_maps(const vtm_split_t* split, int32_t r, int32_t Ns, int32_t Nd, int32_t Bp,
                                const uint64_t* keys_dev, const int32_t* edge_dev, const int32_t* rank_dev,
                                const int32_t* mu_in_dev, const int32_t* pi_in_dev, int32_t pi_offset,
                                int32_t N0, int32_t* mu_out_dev, int32_t* pi_out_dev, void* stream_) {
  using namespace vtm;
  Split sp;
  int rc = make_split(split, &sp);
  if (rc) return rc;
  if (sp.glob_len_dev) return VTM_E_SPLIT;   // device counts: vtm_compose_maps_dev
  if (!mu_out_dev || !pi_out_dev) return VTM_E_NULL;
  if (Ns > 0 && (!keys_dev || !edge_dev || !rank_dev)) return VTM_E_NULL;   // Ns == 0: nothing was matched
  if (sp.Ns != Ns || sp.Nd != Nd || r < 0 || r > Ns || Bp <= 0 || N0 <= 0 || Nd <= 0) return VTM_E_SHAPE;
  if (!pi_in_dev && N0 + pi_offset > sp.N) return VTM_E_SHAPE;
  const int Lnext = (Ns - r) + Nd;
  const int n_iter = Lnext > N0 ? Lnext : N0;
  dim3 grid((n_iter + 255) / 256, Bp);
  compose_maps_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream_)>>>(
      sp, r, Bp, reinterpret_cast<const unsigned long long*>(keys_dev), edge_dev, rank_dev, mu_in_dev,
      pi_in_dev, pi_offset, N0, mu_out_dev, pi_out_dev);
  return launch_rc();
}

extern "C" int vtm_compose_maps_dev(const vtm_split_t* split, const int32_t* counts_dev, int32_t Bp,
                                    const uint64_t* keys_dev, const int32_t* edge_dev, const int32_t* rank_dev,
                                    const int32_t* pi_in_dev, int32_t N0, int32_t* mu_out_dev, int32_t* pi_out_dev,
                                    void* stream_) {
  using namespace vtm;
  Split sp;
  int rc = make_split(split, &sp);
  if (rc) return rc;
  if (!sp.glob_len_dev) return VTM_E_SPLIT;
  if (!counts_dev || !keys_dev || !edge_dev || !rank_dev || !mu_out_dev || !pi_out_dev) return VTM_E_NULL;
  if (Bp <= 0 || N0 <= 0 || (!pi_in_dev && N0 > sp.N)) return VTM_E_SHAPE;
  const int n_iter = sp.N > N0 ? sp.N : N0;     // sp.N = src_len + gcap bounds the merged length
  dim3 grid((n_iter + 255) / 256, Bp);
  compose_maps_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream_)>>>(
      sp, 0, Bp, reinterpret_cast<const unsigned long long*>(keys_dev), edge_dev, rank_dev, nullptr, pi_in_dev, 0, N0,
      mu_out_dev, pi_out_dev, counts_dev);
  return launch_rc();
}

__global__ void split_counts_dev_kernel(vtm::Split sp, double ratio, int* __restrict__ counts) {
  vtm::resolve_split<true>(sp);
  // vtm_merge_count on the device: Python's int(Ns * ratio) in double, then min(Ns, .)
  long long r = static_cast<long long>(trunc(static_cast<double>(sp.Ns) * ratio));
  if (r > sp.Ns) r = sp.Ns;
  counts[0] = sp.Ns;
  counts[1] = sp.Nd;
  counts[2] = static_cast<int>(r);
  counts[3] = sp.Ns - static_cast<int>(r) + sp.Nd;
}

extern "C" int vtm_split_counts_dev(const vtm_split_t* split, double ratio, int32_t* counts_dev, void* stream_) {
  using namespace vtm;
  Split sp;
  int rc = make_split(split, &sp);
  if (rc) return rc;
  if (!sp.glob_len_dev) return VTM_E_SPLIT;
  if (!counts_dev) return VTM_E_NULL;
  if (!(ratio >= 0.0)) return VTM_E_SHAPE;
  split_counts_dev_kernel<<<1, 1, 0, static_cast<cudaStream_t>(stream_)>>>(sp, ratio, counts_dev);
  return launch_rc();
}

extern "C" int vtm_decode_match(const uint64_t* keys_dev, const int32_t* edge_dev, int32_t Bp, int32_t Ns,
                                int32_t Nd, int32_t r, int64_t* unm_idx_dev, int64_t* src_idx_dev,
                                int64_t* dst_idx_dev, uint16_t* node_max_dev, int64_t* node_idx_dev,
                                void* stream_) {
  using namespace vtm;
  if (!keys_dev || !edge_dev) return VTM_E_NULL;
  if (Bp <= 0 || Ns <= 0 || Nd <= 0 || r < 0 || r > Ns) return VTM_E_SHAPE;
  dim3 grid((Ns + 255) / 256, Bp);
  decode_match_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream_)>>>(
      reinterpret_cast<const unsigned long long*>(keys_dev), edge_dev, Ns, Nd, r,
      reinterpret_cast<long long*>(unm_idx_dev), reinterpret_cast<long long*>(src_idx_dev),
      reinterpret_cast<long long*>(dst_idx_dev), node_max_dev, reinterpret_cast<long long*>(node_idx_dev));
  return launch_rc();
}
