// Host/device helpers shared by all translation units: the src/dst split algebra of
// vidtome/merge.py:41-74 and :371-379 in closed form, launch checking, and TMA descriptor creation
// through a runtime-resolved driver entry point (the library never links libcuda, so it loads on a
// machine without a driver and fails only when a compute entry point is called).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/vidtome_b200.h"

namespace vtm {

// Device-side copy of vtm_split_t plus derived counts.
// A mode-1 split with a device coin is stored as the mode-0 split it equals: two "frames" of src_len tokens, stride 2,
// no carried tokens, and the coin picks the dst frame (randf = 1: dst = [src_len, N); randf = 0: dst = [0, src_len)).
// The position algebra below then serves it unchanged.
struct Split {
  int mode, N, unm_pre, F, tnum, stride, randf, src_len;
  int nd_frames;  // local: number of dst frames = #{f in [0,F): f % stride == randf}
  int Ns, Nd;
  const int32_t* randf_dev;  // device-resident randf (NULL = the value above); see resolve_split()
  const float* coin_dev;     // device-resident global coin (NULL = no swap)
  float coin_floor;          // the largest float <= coin_threshold: for a float c, c > coin_floor <=> c > coin_threshold
  // mode 2 (device counts): src_len = L local rows, the global set's length is *glob_len_dev (<= gcap); randf = 1 when the
  // local half is src.  On the host N, Ns and Nd hold capacities (src_len + gcap, cap, cap); resolve_split sets them.
  const int32_t* glob_len_dev;
  int gcap;
  int cap;                   // mode 2: max(src_len, gcap), the row stride of the src / dst buffers (0 in other modes)
};

// Kernels call this first: with a device-resident draw, fetch it (the counts do not depend on it, make_split).
// The coin decides as the host path decides, `float(coin) > global_rand` in double precision (see coin_floor).
// DC: the kernel serves device-count (mode 2) splits; without it that code is compiled out, so the kernels that never see
// one keep their register budgets.
template <bool DC = false>
__device__ __forceinline__ void resolve_split(Split& s) {
  if (s.randf_dev) s.randf = __ldg(s.randf_dev);
  if (s.coin_dev) s.randf = __ldg(s.coin_dev) > s.coin_floor ? 1 : 0;
  if (DC && s.glob_len_dev) {
    const int lg = __ldg(s.glob_len_dev);
    s.N = s.src_len + lg;
    s.Ns = s.randf ? s.src_len : lg;
    s.Nd = s.randf ? lg : s.src_len;
  }
}

__host__ inline int make_split(const vtm_split_t* s, Split* o) {
  if (!s) return VTM_E_NULL;
  o->mode = s->mode; o->N = s->N; o->unm_pre = s->unm_pre; o->F = s->F; o->tnum = s->tnum;
  o->stride = s->stride; o->randf = s->randf; o->src_len = s->src_len; o->nd_frames = 0;
  o->randf_dev = s->mode == 0 ? s->randf_dev : nullptr;
  o->coin_dev = s->mode == 1 || s->mode == 2 ? s->coin_dev : nullptr;
  o->glob_len_dev = nullptr; o->gcap = 0; o->cap = 0;
  // round the threshold down to a float, so that the kernels compare in fp32 and decide exactly as the double
  // comparison does (a NaN threshold stays NaN: never greater, as in double)
  o->coin_floor = static_cast<float>(s->coin_threshold);
  if (static_cast<double>(o->coin_floor) > s->coin_threshold) o->coin_floor = nextafterf(o->coin_floor, -INFINITY);
  if (s->N <= 0) return VTM_E_SPLIT;
  if (s->mode == 0) {
    if (o->randf_dev) {
      // the draw stays on the device: the counts below must not depend on it
      if (s->stride <= 0 || s->F <= 0 || s->F % s->stride != 0) return VTM_E_SPLIT;
      o->randf = 0;
    }
    if (s->F <= 0 || s->tnum <= 0 || s->stride <= 0 || s->stride > s->F || o->randf < 0 ||
        o->randf >= s->stride || s->unm_pre < 0)
      return VTM_E_SPLIT;
    // merge.py:43 tnum = (N - unm_pre) // F; the index buffer covers all N - unm_pre positions and
    // the frame id is pos // tnum (merge.py:59), so N - unm_pre must be exactly F * tnum.
    if ((long long)s->F * s->tnum != (long long)s->N - s->unm_pre) return VTM_E_SPLIT;
    o->nd_frames = (s->F - o->randf + s->stride - 1) / s->stride;
    o->Nd = o->nd_frames * s->tnum + s->unm_pre;
    o->Ns = s->N - o->Nd;
  } else if (s->mode == 1) {
    if (s->src_len < 0 || s->src_len > s->N) return VTM_E_SPLIT;
    if (o->coin_dev) {
      // the coin stays on the device: both halves must be equally long, so that swapping them changes no count
      if ((long long)s->N != 2LL * s->src_len || s->src_len == 0) return VTM_E_SPLIT;
      o->mode = 0; o->unm_pre = 0; o->F = 2; o->tnum = s->src_len; o->stride = 2;
      o->randf = 1;   // [src | dst] until resolve_split reads the coin
      o->nd_frames = 1;
    }
    o->Ns = s->src_len;
    o->Nd = s->N - s->src_len;
  } else if (s->mode == 2) {
    // the tail fields exist only in this mode (modes 0 and 1 may pass the shorter form of the struct)
    if (!s->coin_dev || !s->glob_len_dev || s->src_len <= 0 || s->glob_cap <= 0 ||
        (long long)s->N != (long long)s->src_len + s->glob_cap)
      return VTM_E_SPLIT;
    o->glob_len_dev = s->glob_len_dev;
    o->gcap = s->glob_cap;
    o->cap = s->src_len > s->glob_cap ? s->src_len : s->glob_cap;
    o->randf = 1;
    o->Ns = o->cap;
    o->Nd = o->cap;
  } else {
    return VTM_E_SPLIT;
  }
  return VTM_OK;
}

// position (in the level's sequence) of src token i  — `a_idx[i]`, merge.py:63 / :375
template <bool DC = false>
__host__ __device__ __forceinline__ int src_pos(const Split& s, int i) {
  if (s.mode == 1) return i;
  if (DC && s.mode == 2) return s.randf ? i : s.src_len + i;
  const int q = i / s.tnum, t = i - q * s.tnum;        // q-th src frame
  const int g = q / (s.stride - 1), w = q - g * (s.stride - 1);
  const int f = g * s.stride + (w < s.randf ? w : w + 1);
  return s.unm_pre + f * s.tnum + t;
}
// position of dst token j — `b_idx[j]`, merge.py:64-69 (dst frames then the unm_pre carried tokens) / :376
template <bool DC = false>
__host__ __device__ __forceinline__ int dst_pos(const Split& s, int j) {
  if (s.mode == 1) return s.src_len + j;
  if (DC && s.mode == 2) return s.randf ? s.src_len + j : j;
  const int nf = s.nd_frames * s.tnum;
  if (j >= nf) return j - nf;
  const int q = j / s.tnum, t = j - q * s.tnum;
  return s.unm_pre + (q * s.stride + s.randf) * s.tnum + t;
}
// inverse: position -> (is_dst, index within src or dst)
template <bool DC = false>
__host__ __device__ __forceinline__ bool pos_to_part(const Split& s, int p, int* idx) {
  if (s.mode == 1) {
    if (p < s.src_len) { *idx = p; return false; }
    *idx = p - s.src_len; return true;
  }
  if (DC && s.mode == 2) {   // local rows [0, src_len) are src when randf == 1, global rows [src_len, N) the other half
    const bool local = p < s.src_len;
    *idx = local ? p : p - s.src_len;
    return local != (s.randf != 0);
  }
  if (p < s.unm_pre) { *idx = s.nd_frames * s.tnum + p; return true; }
  const int pp = p - s.unm_pre;
  const int f = pp / s.tnum, t = pp - f * s.tnum;
  const int g = f / s.stride, w = f - g * s.stride;
  if (w == s.randf) { *idx = g * s.tnum + t; return true; }
  const int ord = g * (s.stride - 1) + (w < s.randf ? w : w - 1);
  *idx = ord * s.tnum + t;
  return false;
}

inline int cuda_rc(cudaError_t e) { return e == cudaSuccess ? VTM_OK : static_cast<int>(e); }
inline int launch_rc() { return cuda_rc(cudaGetLastError()); }

// ---- TMA descriptor (cuTensorMapEncodeTiled resolved at run time; no libcuda link dependency)
typedef CUresult (*PFN_tmapEncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                        const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                        const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                        CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline PFN_tmapEncodeTiled get_tmap_encode() {
  // Resolved once per process (the answer cannot change); immutable afterwards, so the entry points stay re-entrant.
  static const PFN_tmapEncodeTiled cached = [] {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      return static_cast<PFN_tmapEncodeTiled>(nullptr);
    return reinterpret_cast<PFN_tmapEncodeTiled>(fn);
  }();
  if (cached) return cached;
  // not resolvable at first use (no driver yet): try again so that a later call can succeed
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) != cudaSuccess ||
      q != cudaDriverEntryPointSuccess)
    return nullptr;
  return reinterpret_cast<PFN_tmapEncodeTiled>(fn);
}

// Number of SMs of the current device; looked up once per device ordinal (immutable afterwards).
inline int cached_sm_count(int* sms) {
  static int table[64];          // 0 = unknown; written once per slot with the same value by any thread
  int dev = 0;
  int rc = cuda_rc(cudaGetDevice(&dev));
  if (rc) return rc;
  if (dev >= 0 && dev < 64 && table[dev] > 0) { *sms = table[dev]; return VTM_OK; }
  int n = 0;
  rc = cuda_rc(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev));
  if (rc) return rc;
  if (dev >= 0 && dev < 64) table[dev] = n;
  *sms = n;
  return VTM_OK;
}

// fp16 tensor [d2][d1][d0] (d0 contiguous), row pitch ld1 elements, slab pitch ld2 elements; box
// {b0, b1, 1}; 128-byte swizzle; out-of-bounds elements read as zero.
inline int make_tmap_3d_f16(CUtensorMap* m, const void* base, uint64_t d0, uint64_t d1, uint64_t d2,
                            uint64_t ld1, uint64_t ld2, uint32_t b0, uint32_t b1) {
  PFN_tmapEncodeTiled enc = get_tmap_encode();
  if (!enc) return VTM_E_DRIVER;
  cuuint64_t dims[3] = {d0, d1, d2};
  cuuint64_t strides[2] = {ld1 * 2, ld2 * 2};
  cuuint32_t box[3] = {b0, b1, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(base), dims, strides, box,
                   estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? VTM_OK : 100000 + static_cast<int>(r);
}

}  // namespace vtm
