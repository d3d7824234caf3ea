/*
 * vidtome_b200 — C-ABI of the H100-native (sm_90a) VidToMe cross-frame token-merge hot path.
 *
 * The reference (lixirui142/VidToMe) is pure Python/PyTorch and has no FFI of its own; every entry
 * point below replaces a span of torch calls in the reference and cites it (file:line relative to the
 * reference tree).  The Python host side (vidtome_b200/merge.py, patch.py) binds these through
 * ctypes exactly as INTEGRATION.md shows; nothing here takes or returns a torch type.
 *
 * Conventions (all entry points):
 *   - every pointer named *_dev is a device pointer (tensor.data_ptr()); `stream` is a cudaStream_t
 *     passed as void* (torch.cuda.current_stream().cuda_stream);
 *   - token matrices are fp16, row-major, rows of C contiguous halfs, C % 8 == 0, 16-byte aligned;
 *   - index maps are int32; "batch stride 0" means one map shared by all samples (align_batch);
 *   - alignment, where an entry point below states none: GEMM operands (A, W, bias, resid, D, LoRA down / up), the
 *     attention entry points' x, ctx, weights, bias, resid and y, and every workspace are 16-byte aligned (they are read
 *     through TMA tensor maps or 16-byte vector accesses); row strides (ldd, ldr, K, C) are multiples of 8 halfs.
 *     Index maps, keys and the other int32 / int64 / fp32 buffers are aligned to their element size.  Results do not
 *     depend on where a buffer sits beyond that, nor on what a workspace held before the call, except where stated;
 *   - the functions never allocate, never synchronise the stream, and never throw; the only process-wide
 *     state is a handful of write-once memoised lookups (driver entry point, SM count, per-kernel shared-memory opt-in
 *     and occupancy), immutable after first use, so calls are re-entrant across streams and devices;
 *   - return value: 0 = ok, <0 = bad argument (VTM_E_*), >0 = a cudaError_t / CUresult reported by
 *     the launch.  There is no CPU fallback: without a CUDA device the compute entry points return
 *     the CUDA error of the failed launch.
 */
#ifndef VIDTOME_B200_H_
#define VIDTOME_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VTM_VERSION 100 /* 0.1.0 */

#define VTM_OK 0
#define VTM_E_NULL (-1)   /* required pointer is NULL */
#define VTM_E_SHAPE (-2)  /* size / divisibility constraint violated */
#define VTM_E_SPLIT (-3)  /* inconsistent vtm_split_t */
#define VTM_E_WS (-4)     /* workspace too small */
#define VTM_E_DRIVER (-5) /* CUDA driver entry point (cuTensorMapEncodeTiled) unavailable */
#define VTM_E_UNSUPPORTED (-6) /* configuration not supported by this build of the kernel */

/*
 * How one matching level partitions its token sequence (length N) into src and dst.
 *   mode 0 (local, random target frame) — bipartite_soft_matching_randframe, vidtome/merge.py:41-74:
 *     sequence = [unm_pre carried tokens | F frames of tnum tokens]; a frame f is dst iff
 *     f % stride == randf; dst = those frames (ascending) followed by the unm_pre carried tokens;
 *     src = the remaining frames (ascending).  stride = min(target_stride, F) (merge.py:55),
 *     randf is the torch.randint value (merge.py:56-57): either drawn to the host (`randf`) or left on the
 *     device (`randf_dev` != NULL: the kernels read *randf_dev, and `randf` is ignored).  The device form lets
 *     a whole denoising step be captured in a CUDA graph whose replays draw fresh values; it requires
 *     F % stride == 0, so that the src / dst counts do not depend on the draw (else VTM_E_SPLIT).
 *   mode 1 (global, prefix/suffix) — bipartite_soft_matching_2s, vidtome/merge.py:371-379:
 *     src = positions [0, src_len), dst = positions [src_len, N).
 *     With `coin_dev` != NULL the global stage's coin (vidtome/patch.py:62, `torch.rand(1) > global_rand`) stays on the
 *     device: the sequence is stored as [local tokens (first src_len rows) | global tokens (the other N - src_len)],
 *     and the kernels compare the fp32 draw *coin_dev in fp32 against `coin_threshold` rounded to the nearest float,
 *     as torch compares an fp32 tensor with a Python float (a draw equal to fp32(global_rand) is never greater):
 *       coin > threshold:     src = [0, src_len), dst = [src_len, N)  (the reference's [local | global], patch.py:63-66);
 *       otherwise:            src = [src_len, N), dst = [0, src_len)  (its [global | local], patch.py:68-71, with
 *                             positions numbered in storage order).
 *     Src row i and dst row j name the same tokens as in the reference either way.  Requires N == 2 * src_len, so
 *     that no count depends on the draw (else VTM_E_SPLIT).
 *   mode 2 (global, device counts) — the mode-1 coin split for token sets of different lengths, where the counts
 *     depend on the draw: the sequence is stored as [local (src_len rows, host-known) | global (*glob_len_dev rows, at
 *     most glob_cap)], N == src_len + glob_cap is its capacity, and coin_dev / coin_threshold pick the src half as in
 *     mode 1 (coin > threshold: src = local; otherwise src = global; positions in storage order).  Ns, Nd, r and the
 *     merged length live on the device (vtm_split_counts_dev) and the *_dev entry points below read them; buffers are
 *     sized for capacity (vtm_split_counts returns cap = max(src_len, glob_cap) for both counts).  The fields
 *     glob_len_dev and glob_cap are read only in this mode, so a caller may pass the 56-byte form of the struct
 *     for modes 0 and 1.
 */
typedef struct vtm_split {
  int32_t mode;
  int32_t N;
  int32_t unm_pre;
  int32_t F;
  int32_t tnum;
  int32_t stride;
  int32_t randf;
  int32_t src_len;
  const int32_t* randf_dev; /* optional device-resident randf (mode 0), NULL = use `randf` */
  const float* coin_dev;    /* optional device-resident global coin (mode 1), NULL = plain prefix split */
  double coin_threshold;    /* global_rand: the halves swap roles when !(coin > (float)coin_threshold) */
  const int32_t* glob_len_dev; /* mode 2: device-resident length of the global set, 1 <= *glob_len_dev <= glob_cap */
  int32_t glob_cap;            /* mode 2: capacity of the global set */
} vtm_split_t;

/* Length of the device counts record written by vtm_split_counts_dev: {Ns, Nd, r, M = Ns - r + Nd}. */
#define VTM_COUNTS_LEN 4

/* Library version (VTM_VERSION).  Pure host. */
int vtm_version(void);

/* Human-readable text for a return code of this library (negative codes) or "cuda error". */
const char* vtm_error_string(int code);

/* Host helper: number of src / dst tokens of a split (merge.py:63-71 `a_idx`, `b_idx`, `num_dst`;
 * merge.py:375-379 for mode 1).  Pure host, no CUDA. */
int vtm_split_counts(const vtm_split_t* split, int32_t* num_src, int32_t* num_dst);

/* Host helper: r = min(Ns, int(Ns * ratio)) with Python-double truncation (merge.py:90, :395). */
int32_t vtm_merge_count(int32_t num_src, double ratio);

/* Device counts of a mode-2 split: one tiny kernel resolves the coin and the global length and writes
 * counts_dev[0..3] = {Ns, Nd, r = min(Ns, int(Ns * ratio)) in double as vtm_merge_count, M = Ns - r + Nd}.
 * Nothing is read back to the host.  Other modes: VTM_E_SPLIT. */
int vtm_split_counts_dev(const vtm_split_t* split, double ratio, int32_t* counts_dev, void* stream);

/*
 * K0 — row-normalise and split.  Replaces `metric / metric.norm(dim=-1, keepdim=True)` followed by
 * `split(metric)` (two torch.gather calls), vidtome/merge.py:76-85 and :381-390.
 *   x_dev        [B, *, C] fp16 original tokens; sample stride x_batch_stride elements
 *   rowmap_dev   [B'|1, split->N] int32: position in this level's sequence -> row of x (NULL = identity);
 *                rowmap_batch_stride = 0 shares one map across samples
 *   a_out_dev    [B, Ns, C] fp16 normalised src rows;  b_out_dev [B, Nd, C] fp16 normalised dst rows
 * Normalisation follows torch half semantics: fp32 sum of squares -> sqrt -> round to fp16 -> each
 * element fp16(float(x) / float(norm)); no epsilon (merge.py:84).
 */
int vtm_normalize_split(const void* x_dev, int64_t x_batch_stride, const int32_t* rowmap_dev,
                        int64_t rowmap_batch_stride, const vtm_split_t* split, int32_t B, int32_t C,
                        void* a_out_dev, void* b_out_dev, void* stream);

/*
 * K0 with the block's LayerNorm fused in front: rows are read from the RAW hidden states, normalised with
 * (ln_weight, ln_bias, ln_eps) exactly as `self.norm1(hidden_states)` does (vidtome/patch.py:146; torch
 * half semantics: fp32 statistics, y = gamma * (rstd * (x - mean)) + beta rounded to fp16) and then handled
 * as in vtm_normalize_split.  norm1's output is never written to memory.  ln_weight_dev == NULL disables
 * the LayerNorm (== vtm_normalize_split); ln_bias_dev may be NULL.
 */
int vtm_normalize_split_ln(const void* x_dev, int64_t x_batch_stride, const int32_t* rowmap_dev,
                           int64_t rowmap_batch_stride, const vtm_split_t* split, int32_t B, int32_t C,
                           const void* ln_weight_dev, const void* ln_bias_dev, float ln_eps, void* a_out_dev,
                           void* b_out_dev, void* stream);

/*
 * KA — fused similarity + row arg-max on wgmma tensor cores.  Replaces
 * `scores = a @ b.transpose(-1, -2)` and `scores.max(dim=-1)` (vidtome/merge.py:87,112 and :392,416)
 * and, with align_batch != 0, `torch.cat([*scores], dim=-1)` + max (merge.py:93-97, :398-401).
 * The Ns x Nd score matrix is never written: accumulators live on chip, are rounded to fp16 exactly
 * as the reference's fp16 `scores` tensor is, and reduced per row with first-index tie breaking.
 *   a_dev [B, Ns, C], b_dev [B, Nd, C] fp16 (outputs of vtm_normalize_split)
 *   keys_out_dev [B' , Ns] uint64, B' = 1 if align_batch else B.  Packed result per src row:
 *       bits 32..47  order-preserving image of the fp16 row maximum (vtm_key_score())
 *       bits  0..31  0xFFFFFFFF - arg, arg = dst index j, or b*Nd + j when align_batch
 *   The buffer is zeroed by this call (cudaMemsetAsync on `stream`) before the kernel runs.
 * Non-finite scores: a NaN score never wins, so a src row with a NaN entry publishes nothing (its key stays 0) and a
 * NaN dst column is never the arg; a score that rounds to +inf competes as +inf.  A row whose every score is -inf
 * publishes nothing either (key 0), where torch's max gives (-inf, index 0).  Neither happens for the unit rows K0
 * writes: their scores are finite and at most about 1 in magnitude.
 */
int vtm_sim_argmax(const void* a_dev, const void* b_dev, int32_t B, int32_t Ns, int32_t Nd,
                   int32_t C, int32_t align_batch, uint64_t* keys_out_dev, void* stream);

/* Debug/verification twin of KA on CUDA cores (one thread per src row, sequential fp32 FMA over K
 * in index order).  Same outputs; used by tests to cross-check KA at sizes the CPU oracle cannot
 * reach.  Not used by the product path. */
int vtm_sim_argmax_simt(const void* a_dev, const void* b_dev, int32_t B, int32_t Ns, int32_t Nd,
                        int32_t C, int32_t align_batch, uint64_t* keys_out_dev, void* stream);

/* KA with device counts (mode-2 splits): a_dev [B, ns_cap, C] and b_dev [B, nd_cap, C] as vtm_normalize_split writes
 * them for such a split; Ns = counts_dev[0] and Nd = counts_dev[1] are read on the device.  Src rows >= Ns publish
 * nothing and dst columns >= Nd take no part; keys_out_dev is [B', ns_cap] (row stride ns_cap), zeroed first.  The keys
 * of the first Ns rows equal those of vtm_sim_argmax called with the same counts as host values.  The SIMT twin has
 * no such path. */
int vtm_sim_argmax_dev(const void* a_dev, const void* b_dev, int32_t B, int32_t ns_cap, int32_t nd_cap, int32_t C,
                       int32_t align_batch, const int32_t* counts_dev, uint64_t* keys_out_dev, void* stream);

/* Unpack helpers for KA keys (pure host; the same bit rules are used on the device). */
uint16_t vtm_key_score_half_bits(uint64_t key); /* fp16 bit pattern of the row maximum */
uint32_t vtm_key_arg(uint64_t key);             /* arg as defined above */

/*
 * KB1 — stable descending order of the row maxima.  Replaces `node_max.argsort(dim=-1,
 * descending=True)` (vidtome/merge.py:98,113,402,417) with stable semantics (ties -> lower src row
 * first), which is what torch's CUDA radix path produces and what the oracle pins.
 *   keys_dev  [Bp, Ns] uint64 from KA
 *   edge_dev  [Bp, Ns] int32: edge[k] = src row with the k-th largest maximum
 *   rank_dev  [Bp, Ns] int32: rank[edge[k]] = k
 *   ws_dev    workspace of at least vtm_topr_workspace_bytes(Bp, Ns) bytes
 */
size_t vtm_topr_workspace_bytes(int32_t Bp, int32_t Ns);
int vtm_topr_sort(const uint64_t* keys_dev, int32_t Bp, int32_t Ns, int32_t* edge_dev,
                  int32_t* rank_dev, void* ws_dev, size_t ws_bytes, void* stream);

/*
 * KB2 — apply one level's match to the composed index maps.  Replaces the index bookkeeping of the
 * merge / unmerge closures (vidtome/merge.py:115-155, :419-459) and their composition through
 * func_warper (vidtome/patch.py:84-85): in "replace" mode every level is a row gather, so the whole
 * merge is one gather `merged[i] = x[mu[i]]` and the whole unmerge is one gather `out[p] = y[pi[p]]`.
 *   split, r, Ns, Nd      this level (r = vtm_merge_count)
 *   keys_dev/edge_dev/rank_dev [Bp, Ns] from KA / KB1
 *   mu_in_dev  [Bp, split->N] int32 position -> row of the level-0 token table (NULL = identity)
 *   pi_in_dev  [Bp, N0] int32 level-0 position -> position in this level's sequence (NULL = identity,
 *              requires N0 == split->N); pi_offset is added to every pi_in entry first (global stage:
 *              the local tokens sit at [pi_offset, pi_offset + L) of the concatenated sequence)
 *   mu_out_dev [Bp, (Ns - r) + Nd] int32;  pi_out_dev [Bp, N0] int32
 * Merged sequence order is [unmerged src (edge[r:]) | dst], as merge.py:133 `cat([unm, dst])`.
 */
int vtm_compose_maps(const vtm_split_t* split, int32_t r, int32_t Ns, int32_t Nd, int32_t Bp,
                     const uint64_t* keys_dev, const int32_t* edge_dev, const int32_t* rank_dev,
                     const int32_t* mu_in_dev, const int32_t* pi_in_dev, int32_t pi_offset, int32_t N0,
                     int32_t* mu_out_dev, int32_t* pi_out_dev, void* stream);

/* KB1 / KB2 with device counts (mode-2 splits).  keys, edge and rank are [Bp, ns_cap] with row stride ns_cap and only
 * their first counts_dev[0] entries per row take part.  vtm_compose_maps_dev reads Ns, Nd and r from counts_dev; mu_out is
 * [Bp, split->N] (its first M entries are meaningful), pi_out is [Bp, N0]; with pi_in_dev == NULL only the first
 * src_len + *glob_len_dev entries of pi_out are written.  mu_in_dev is not supported (NULL). */
int vtm_topr_sort_dev(const uint64_t* keys_dev, int32_t Bp, int32_t ns_cap, const int32_t* counts_dev, int32_t* edge_dev,
                      int32_t* rank_dev, void* ws_dev, size_t ws_bytes, void* stream);
int vtm_compose_maps_dev(const vtm_split_t* split, const int32_t* counts_dev, int32_t Bp, const uint64_t* keys_dev,
                         const int32_t* edge_dev, const int32_t* rank_dev, const int32_t* pi_in_dev, int32_t N0,
                         int32_t* mu_out_dev, int32_t* pi_out_dev, void* stream);

/* Decode KA/KB1 results into the reference's own index tensors (int64, as torch returns them):
 * unm_idx = edge[r:], src_idx = edge[:r], dst_idx = node_idx[src_idx] (% Nd when align_batch)
 * (vidtome/merge.py:100-108,115-117).  node_max_dev (fp16 bits) / node_idx_dev may be NULL. */
int vtm_decode_match(const uint64_t* keys_dev, const int32_t* edge_dev, int32_t Bp, int32_t Ns,
                     int32_t Nd, int32_t r, int64_t* unm_idx_dev, int64_t* src_idx_dev,
                     int64_t* dst_idx_dev, uint16_t* node_max_dev, int64_t* node_idx_dev, void* stream);

/*
 * KC — merge gather: y[b, i, :] = x[b, map[b, i], :].  Replaces merge() of every level
 * (vidtome/merge.py:119-133, :423-437) composed by func_warper (patch.py:84), in one pass.
 */
int vtm_gather_rows(const void* x_dev, int64_t x_batch_stride, const int32_t* map_dev,
                    int64_t map_batch_stride, int32_t B, int32_t L, int32_t C, void* y_dev,
                    int64_t y_batch_stride, void* stream);

/*
 * KC as the producer of the global-token exchange (SURVEY.md §8e, the all-gather variant of vidtome/patch.py:59-82
 * sharded one chunk per GPU): same as vtm_gather_rows_ln, and every output row is ALSO stored to n_peers (<= 8)
 * further destinations `peer_y_devs[i]` — buffers of the same layout in other GPUs' memory, peer-mapped into this
 * process (NVLink P2P; e.g. torch symmetric memory).  The merged tokens reach all ranks in the pass that creates
 * them; the caller only adds a barrier before reading the peers' contributions.  peer_y_devs is a HOST array.
 */
int vtm_gather_rows_peers(const void* x_dev, int64_t x_batch_stride, const int32_t* map_dev,
                          int64_t map_batch_stride, int32_t B, int32_t L, int32_t C, const void* ln_weight_dev,
                          const void* ln_bias_dev, float ln_eps, void* y_dev, int64_t y_batch_stride,
                          void* const* peer_y_devs, int32_t n_peers, void* stream);

/* KC with norm1 fused: y[b, i, :] = LayerNorm(x[b, map[b, i], :]) — the merged tokens that feed attn1,
 * computed from the raw hidden states (only the L kept rows are ever normalised). */
int vtm_gather_rows_ln(const void* x_dev, int64_t x_batch_stride, const int32_t* map_dev,
                       int64_t map_batch_stride, int32_t B, int32_t L, int32_t C, const void* ln_weight_dev,
                       const void* ln_bias_dev, float ln_eps, void* y_dev, int64_t y_batch_stride, void* stream);

/* KC with a device row count: rows i < *len_dev are gathered as in vtm_gather_rows, rows [*len_dev, L_cap) are written
 * as zeros (so that nothing stale or non-finite reaches a kernel that runs over capacity). */
int vtm_gather_rows_dev(const void* x_dev, int64_t x_batch_stride, const int32_t* map_dev, int64_t map_batch_stride,
                        int32_t B, int32_t L_cap, int32_t C, const int32_t* len_dev, void* y_dev, int64_t y_batch_stride,
                        void* stream);

/*
 * Merge with a reduction — the non-"replace" modes of the merge closure, vidtome/merge.py:126-131:
 * `dst.scatter_reduce(-2, dst_idx, src[src_idx], reduce=mode, include_self=True)` followed by `cat([unm, dst])`.
 *   mode: 1 = "mean", 2 = "sum", 3 = "amax", 4 = "amin" ("prod" is not implemented: VTM_E_UNSUPPORTED)
 *   x_dev [B, split->N, C] fp16 (the tensor being merged; finite values), keys/edge [Bp, Ns] from KA / KB1, r as in KB2
 *   y_dev [B, (Ns - r) + Nd, C] fp16;  ws_dev: vtm_merge_reduce_workspace_bytes(B, Nd, C) bytes
 * Sums are exact and order independent (int64 fixed-point accumulators, value * 2^24) and rounded once; the mean is
 * fp16(float(sum) / float(count)) as torch computes it.  The reference accumulates in fp16 (CPU: index order; CUDA:
 * atomics in arbitrary order) and therefore agrees bit for bit only where its partial sums are exact.
 * No caller in the reference passes a mode; a reduction is not a row gather, so this is an operator-API entry and
 * not part of the composed per-block plan.
 */
size_t vtm_merge_reduce_workspace_bytes(int32_t B, int32_t Nd, int32_t C);
int vtm_merge_reduce(const void* x_dev, int64_t x_batch_stride, const vtm_split_t* split, int32_t r, int32_t Bp,
                     const uint64_t* keys_dev, const int32_t* edge_dev, int32_t B, int32_t C, int32_t mode,
                     void* y_dev, void* ws_dev, size_t ws_bytes, void* stream);

/*
 * KE — unmerge gather fused with the residual add: out[b, p, :] = y[b, map[b, p], :] + resid[b, p, :].
 * Replaces unmerge() of every level (zeros + 3 scatter_, vidtome/merge.py:135-155, :439-460),
 * split_frame (vidtome/utils.py:37-40) and `attn_output + hidden_states` (vidtome/patch.py:168-169).
 * resid_dev may be NULL (plain unmerge, used by the merge.py-level API).
 */
int vtm_unmerge_add(const void* y_dev, int64_t y_batch_stride, const int32_t* map_dev,
                    int64_t map_batch_stride, const void* resid_dev, int32_t B, int32_t N, int32_t C,
                    void* out_dev, void* stream);

/*
 * KD — merged-token self-attention.  Replaces `self.attn1(merged_tokens)` (vidtome/patch.py:157-162;
 * math restated in the reference at utils/pnp_utils.py:47-95): q,k,v = x Wq^T, x Wk^T, x Wv^T (no bias),
 * per-head softmax(q k^T * scale) v, heads re-joined, y = o Wo^T + bo.
 *   x_dev [B, L, C] fp16; w_qkv_dev [3C, C] fp16 (rows: Wq | Wk | Wv, torch Linear layout);
 *   w_o_dev [C, C] fp16; b_o_dev [C] fp16 (may be NULL); heads * head_dim == C; head_dim % 8 == 0 and head_dim <= 160 (else VTM_E_SHAPE / VTM_E_UNSUPPORTED)
 *   y_dev [B, L, C] fp16; ws_dev workspace of vtm_attention_workspace_bytes(B, L, C, heads) bytes (q/k/v head-major
 *   with rows padded to 64, 128 or 192 halfs for head_dim <= 64, <= 128, <= 160, plus the attention output before the
 *   out projection).
 */
size_t vtm_attention_workspace_bytes(int32_t B, int32_t L, int32_t C, int32_t heads);
int vtm_attention(const void* x_dev, const void* w_qkv_dev, const void* w_o_dev, const void* b_o_dev,
                  int32_t B, int32_t L, int32_t C, int32_t heads, float scale, void* y_dev,
                  void* ws_dev, size_t ws_bytes, void* stream);

/* KD with options.  flags bit 0 (VTM_ATTN_SHARED_QK): PnP's source-sample injection (utils/pnp_utils.py:57-68,87-91: the
 * attention map softmax(q k^T) is computed from sample 0 only and `repeat`ed over the batch): every sample b uses the
 * queries and keys of sample 0 and its own values.  q and k of samples 1..B-1 are not computed (their part of the
 * workspace is left as it was), and the map is computed once for a group of samples.  Other bits must be zero
 * (VTM_E_UNSUPPORTED). */
#define VTM_ATTN_SHARED_QK 1
int vtm_attention_ex(const void* x_dev, const void* w_qkv_dev, const void* w_o_dev, const void* b_o_dev,
                     int32_t B, int32_t L, int32_t C, int32_t heads, float scale, int32_t flags, void* y_dev,
                     void* ws_dev, size_t ws_bytes, void* stream);

/* KD with a device sequence length: x_dev / y_dev are [B, L_cap, C] and the sequence is the first *len_dev rows of each
 * sample (1 <= *len_dev <= L_cap).  The projections run over all L_cap rows (rows are independent; rows past the length
 * must be finite, e.g. the zeros of vtm_gather_rows_dev), the flash kernel reads the length on the device, and rows
 * < *len_dev of y equal those of vtm_attention_ex called with L = *len_dev, bit for bit.  Rows past it are unspecified.
 * Workspace: vtm_attention_workspace_bytes(B, L_cap, C, heads). */
int vtm_attention_dev(const void* x_dev, const void* w_qkv_dev, const void* w_o_dev, const void* b_o_dev,
                      int32_t B, int32_t L_cap, int32_t C, int32_t heads, float scale, int32_t flags,
                      const int32_t* len_dev, void* y_dev, void* ws_dev, size_t ws_bytes, void* stream);

/* Plain wgmma GEMM used by KD's projections, exported for tests and the microbench:
 * D[M, N] = A[M, K] * W[N, K]^T (+ bias[N]), fp16 in, fp32 accumulate, fp16 out.  K % 8 == 0,
 * N % 8 == 0; ldd = row stride of D in elements. */
int vtm_linear_f16(const void* a_dev, const void* w_dev, const void* bias_dev, int32_t M, int32_t N,
                   int32_t K, void* d_dev, int64_t ldd, void* stream);

/*
 * Cross-attention of the patched block.  Replaces `self.attn2(norm2(h), encoder_hidden_states=ctx) + h`
 * (vidtome/patch.py:171-185; diffusers Attention with K/V taken from the text context):
 *   q = x Wq^T, [k | v] = ctx [Wk; Wv]^T (no bias), per-head softmax(q k^T * scale) v, y = o Wo^T + bo (+ resid).
 *   x_dev [B, Lq, C] fp16 (norm2 output); ctx_dev [B, Lk, Cctx] fp16; w_q_dev [C, C]; w_kv_dev [2C, Cctx] (rows Wk | Wv);
 *   w_o_dev [C, C]; b_o_dev [C] or NULL; resid_dev [B, Lq, C] or NULL; y_dev [B, Lq, C].
 *   B counts (sample x frame) items: every item attends to its own Lk context rows.  head_dim % 8 == 0, <= 160.
 */
size_t vtm_cross_attention_workspace_bytes(int32_t B, int32_t Lq, int32_t Lk, int32_t C, int32_t heads);
int vtm_cross_attention(const void* x_dev, const void* ctx_dev, const void* w_q_dev, const void* w_kv_dev,
                        const void* w_o_dev, const void* b_o_dev, const void* resid_dev, int32_t B, int32_t Lq,
                        int32_t Lk, int32_t C, int32_t Cctx, int32_t heads, float scale, void* y_dev, void* ws_dev,
                        size_t ws_bytes, void* stream);

/*
 * Feed-forward of the patched block (vidtome/patch.py:187-199 calls `self.ff(norm3(h))` and adds the residual; the
 * module is diffusers' FeedForward = GEGLU(dim -> 4 dim) -> Dropout -> Linear(4 dim -> dim)) on wgmma:
 *
 * vtm_linear_geglu_f16:  D[M, N/2] = h * gelu(gate) with [h | gate] = A[M, K] * W^T + bias (erf form of gelu, torch's
 *   F.gelu default).  `w_il_dev` [N, K] and `bias_il_dev` [N] hold the projection's rows INTERLEAVED in groups of 32:
 *   rows [64 q, 64 q + 32) = rows [32 q, 32 q + 32) of the value half, rows [64 q + 32, 64 q + 64) = the same rows of the
 *   gate half (so that a value and its gate land in one 64-column accumulator slice).  N % 64 == 0.  Roundings follow torch's
 *   fp16 pipeline: projection -> fp16, gelu(gate) -> fp16, product -> fp16.
 * vtm_linear_residual_f16:  D[M, N] = fp16(fp16(A W^T + bias) + resid[M, N]) — `lin(x) + hidden_states`.
 */
int vtm_linear_geglu_f16(const void* a_dev, const void* w_il_dev, const void* bias_il_dev, int32_t M, int32_t N,
                         int32_t K, void* d_dev, int64_t ldd, void* stream);
int vtm_linear_residual_f16(const void* a_dev, const void* w_dev, const void* bias_dev, const void* resid_dev,
                            int64_t ldr, int32_t M, int32_t N, int32_t K, void* d_dev, int64_t ldd, void* stream);

/*
 * LoRA-adapted projections.  A LoRA layer computes y = x W^T + b + sum_a s_a (x A_a^T) B_a^T (diffusers'
 * LoRACompatibleLinear and peft's lora.Linear, which the reference loads with `pipe.load_lora_weights`, generate.py:93-94).
 * The adapters of a GEMM are stacked into one "down" matrix D [R, K] (the A_a rows) and one "up" matrix U [N, R] (the
 * s_a B_a columns, zero where an adapter does not feed an output), and the library computes
 *     y = fp16([x | T] [W | U]^T + b),   T = fp16(x D^T)
 * i.e. the projection GEMM with R more K steps taken from (T, U): one fp32 accumulation and one final rounding, every
 * epilogue (head split, bias, residual, GEGLU) unchanged.  T is computed into the caller's workspace by one extra launch
 * of the store GEMM (N = R) per adapted GEMM.  A NULL descriptor or R == 0 gives bit for bit the result of the entry
 * point without LoRA.  Nothing allocates or synchronises; every call can be captured in a CUDA graph.
 */
typedef struct vtm_lora_t {
  const void* down_dev;  /* [R, K] fp16: lora_A rows of every active adapter of the GEMM's projections, stacked   */
  const void* up_dev;    /* [N, R] fp16: matching lora_B columns with each adapter's scale folded in, 0 elsewhere */
  int32_t R;             /* total rank, a multiple of 8 (pad with zero rows / columns); 0 = no LoRA               */
} vtm_lora_t;

/* vtm_linear_f16 / vtm_linear_residual_f16 with a LoRA: D[M, N] = fp16(A W^T + T U^T + bias) (resid_dev == NULL), or
 * fp16(fp16(A W^T + T U^T + bias) + resid) with resid [M, ldr].  Workspace: vtm_linear_lora_workspace_bytes(M, R)
 * (T [M, R]; 0 for R == 0, and ws_dev may then be NULL). */
size_t vtm_linear_lora_workspace_bytes(int32_t M, int32_t R);
int vtm_linear_lora_f16(const void* a_dev, const void* w_dev, const void* bias_dev, const void* resid_dev, int64_t ldr,
                        const vtm_lora_t* lora, int32_t M, int32_t N, int32_t K, void* d_dev, int64_t ldd, void* ws_dev,
                        size_t ws_bytes, void* stream);

/* vtm_linear_geglu_f16 with a LoRA on the GEGLU projection: lora->up_dev [N, R] has its rows interleaved in groups of
 * 32 exactly as w_il_dev.  Workspace: vtm_linear_lora_workspace_bytes(M, R). */
int vtm_linear_geglu_lora_f16(const void* a_dev, const void* w_il_dev, const void* bias_il_dev, const vtm_lora_t* lora,
                              int32_t M, int32_t N, int32_t K, void* d_dev, int64_t ldd, void* ws_dev, size_t ws_bytes,
                              void* stream);

/* KD with LoRAs: vtm_attention_ex (len_dev == NULL) or vtm_attention_dev (len_dev != NULL, L = L_cap) with
 *   lora_qkv: the QKV GEMM, D [R, C], U [3C, R] (block-diagonal over the q / k / v row blocks);
 *   lora_o:   to_out[0], D [R, C], U [C, R]; T is computed from the attention output between the flash kernel and the
 *             output projection.
 * Under VTM_ATTN_SHARED_QK q and k take the tail rows of sample 0 and v rows [2C, 3C) of U, as their weights do.
 * Workspace: vtm_attention_lora_workspace_bytes(B, L, C, heads, R_qkv, R_o). */
size_t vtm_attention_lora_workspace_bytes(int32_t B, int32_t L, int32_t C, int32_t heads, int32_t R_qkv, int32_t R_o);
int vtm_attention_lora(const void* x_dev, const void* w_qkv_dev, const void* w_o_dev, const void* b_o_dev,
                       const vtm_lora_t* lora_qkv, const vtm_lora_t* lora_o, int32_t B, int32_t L, int32_t C,
                       int32_t heads, float scale, int32_t flags, const int32_t* len_dev, void* y_dev, void* ws_dev,
                       size_t ws_bytes, void* stream);

/* vtm_cross_attention with LoRAs: lora_q on to_q (D [Rq, C], U [C, Rq], applied to x), lora_kv on to_k / to_v
 * (D [Rkv, Cctx], U [2C, Rkv], applied to the context), lora_o on to_out[0] (D [Ro, C], U [C, Ro]; the residual is
 * added after it as without LoRA).  Workspace: vtm_cross_attention_lora_workspace_bytes(B, Lq, Lk, C, heads, Rq, Rkv, Ro). */
size_t vtm_cross_attention_lora_workspace_bytes(int32_t B, int32_t Lq, int32_t Lk, int32_t C, int32_t heads, int32_t R_q,
                                                int32_t R_kv, int32_t R_o);
int vtm_cross_attention_lora(const void* x_dev, const void* ctx_dev, const void* w_q_dev, const void* w_kv_dev,
                             const void* w_o_dev, const void* b_o_dev, const void* resid_dev, const vtm_lora_t* lora_q,
                             const vtm_lora_t* lora_kv, const vtm_lora_t* lora_o, int32_t B, int32_t Lq, int32_t Lk,
                             int32_t C, int32_t Cctx, int32_t heads, float scale, void* y_dev, void* ws_dev,
                             size_t ws_bytes, void* stream);

/*
 * KT — the residual tail of PnP's feature-injected ResNet (utils/pnp_utils.py:146-162, `register_conv_control`):
 *   out[b] = (shortcut[b] + h[src(b)]) / output_scale_factor
 * with src(b) = b mod n for b in [n, 2n) and [2n, 3n) when `inject` is 1 (the source samples' conv2 output copied over
 * the uncond and cond samples), and src(b) = b otherwise.
 *   h_dev         conv2's output: [num_inputs * n, E] fp16, or only its source samples [n, E] when inject is 1
 *   shortcut_dev  [num_inputs * n, E] fp16: conv_shortcut(input), or the input itself when the block has no shortcut
 *   out_dev       [num_inputs * n, E] fp16;  E = sample_elems = C * H * W (any value); contiguous NCHW tensors
 *   num_inputs    1..3 (VTM_E_UNSUPPORTED otherwise);  inject 0 or 1
 * Rounding is that of torch's CUDA half ops: fp16(float(s) + float(h)), then fp16(float(sum) * (1.0f / osf)) (torch
 * divides a CUDA tensor by a CPU scalar as a multiplication by the fp32 reciprocal).  output_scale_factor must be finite
 * and non-zero (VTM_E_UNSUPPORTED).  Pointers must be 2-byte aligned (VTM_E_SHAPE); 16-byte vectors are used wherever the
 * three streams share their offset from a 16-byte boundary.
 */
int vtm_resnet_tail_f16(const void* h_dev, const void* shortcut_dev, void* out_dev, int32_t n, int32_t num_inputs,
                        int64_t sample_elems, float output_scale_factor, int32_t inject, void* stream);

/*
 * KD with the residual in the out projection — the self-attention of an UNMERGED block, `attn1(norm1(h)) + h`
 * (vidtome/patch.py:157-169 with merge and unmerge = do_nothing; DDIM inversion runs the UNet unpatched,
 * invert.py:117-140):
 *   y = fp16(fp16(o Wo^T + bo) + resid),  o = per-head softmax(q k^T * scale) v,  q,k,v = x Wq^T, x Wk^T, x Wv^T
 *   x_dev [B, L, C] fp16 (norm1's output); resid_dev [B, L, C] fp16 (the block input h, required: VTM_E_NULL);
 *   y_dev [B, L, C] fp16, not overlapping resid_dev.  B counts (sample x frame) items; each item attends only within
 *   its own L rows.  Weights, head_dim limits and LoRA descriptors as vtm_attention_lora (NULL = no adapter); no
 *   shared-q/k injection.  The result equals vtm_attention_ex (or vtm_attention_lora) followed by torch's half add,
 *   bit for bit: the add is the out projection's residual epilogue of vtm_linear_residual_f16.
 *   Workspace: vtm_attention_lora_workspace_bytes(B, L, C, heads, R_qkv, R_o) (vtm_attention_workspace_bytes without
 *   adapters).
 */
int vtm_attention_residual(const void* x_dev, const void* w_qkv_dev, const void* w_o_dev, const void* b_o_dev,
                           const void* resid_dev, const vtm_lora_t* lora_qkv, const vtm_lora_t* lora_o, int32_t B,
                           int32_t L, int32_t C, int32_t heads, float scale, void* y_dev, void* ws_dev,
                           size_t ws_bytes, void* stream);

/*
 * vtm_attention_residual with PnP's source-frame injection, for the self-attention of an unmerged block during PnP
 * generation (utils/pnp_utils.py:57-68, 86-91: `q[:B // num_inputs]`, `k[:B // num_inputs]` and
 * `attn.repeat(num_inputs, 1, 1)` on a batch of [source | uncond | cond] frame items):
 *   flags == 0:                   bit for bit vtm_attention_residual; qk_items is ignored.
 *   flags == VTM_ATTN_SHARED_QK:  item b uses the attention map of item b mod qk_items, i.e. the queries and keys of item
 *                                 b mod qk_items and its own values.  1 <= qk_items and B % qk_items == 0, else
 *                                 VTM_E_SHAPE.  q and k are computed for the first qk_items items only (their part of
 *                                 the workspace for the other items is left as it was).  The result equals, bit for
 *                                 bit, vtm_attention_ex(VTM_ATTN_SHARED_QK) on the items {f, f + qk_items, ...} of each
 *                                 f < qk_items, followed by torch's half add of the residual.
 *   Other flag bits: VTM_E_UNSUPPORTED.  resid_dev == NULL: VTM_E_NULL.  Everything else as vtm_attention_residual,
 *   workspace vtm_attention_lora_workspace_bytes(B, L, C, heads, R_qkv, R_o).  No allocation, no synchronisation:
 *   capturable in a CUDA graph.
 */
int vtm_attention_residual_ex(const void* x_dev, const void* w_qkv_dev, const void* w_o_dev, const void* b_o_dev,
                              const void* resid_dev, const vtm_lora_t* lora_qkv, const vtm_lora_t* lora_o, int32_t B,
                              int32_t L, int32_t C, int32_t heads, float scale, int32_t flags, int32_t qk_items,
                              void* y_dev, void* ws_dev, size_t ws_bytes, void* stream);

/*
 * KI — one DDIM step in place, with its coefficients and trajectory slot read on the device (replaces the update of
 * invert.py:182-211, `pred_next_x(..., inversion=True)`, and stores what invert.py:132-138 saves):
 *   s = *step_dev;  (a, r, c, d) = coef_dev[4 s .. 4 s + 3];  x <- c * ((x - a * eps) * r) + d * eps,  r = 1 / b;
 *   if slot_dev != NULL and 0 <= slot_dev[s] < n_slots:  traj[slot_dev[s]] <- x  (traj_dev [n_slots, n])
 * For inversion a = sigma_prev, b = mu_prev, c = mu, d = sigma; for sampling (generate.py:281-311) a = sigma, b = mu,
 * c = mu_prev, d = sigma_prev.  Because the step is read on the device, one captured
 * CUDA graph serves every step; the caller advances *step_dev.  A step outside [0, n_steps) leaves x unchanged.
 *   x_dev, eps_dev [n] fp16 (any n >= 1), 2-byte aligned (VTM_E_SHAPE); coef_dev [n_steps, 4] fp32, 16-byte aligned;
 *   step_dev, slot_dev int32, 4-byte aligned; slot_dev may be NULL (no trajectory; traj_dev and n_slots are then
 *   ignored), otherwise traj_dev is required (VTM_E_NULL) and n_slots >= 1 (VTM_E_SHAPE).
 * Rounding is that of torch's CUDA half ops on python-float coefficients: each product, difference and sum is computed
 * in fp32 and rounded to fp16, and the division is a multiplication by the reciprocal, which torch computes in double
 * and rounds once to fp32: r = (float)(1.0 / b) in the table reproduces `half_tensor / python_float` bit for bit.
 * 16-byte vectors are used wherever x, eps and the slot share their offset from a 16-byte boundary.
 */
int vtm_ddim_update_f16(void* x_dev, const void* eps_dev, int64_t n, const float* coef_dev, const int32_t* slot_dev,
                        const int32_t* step_dev, int32_t n_steps, void* traj_dev, int32_t n_slots, void* stream);

/*
 * KS — the sampling step's classifier-free guidance combine and DDIM update in one pass, for one chunk
 * (generate.py:274-279, the guidance combine of pred_noise, and generate.py:281-311, pred_next_x with inversion=False):
 *   u = eps[(samples - 2) n ..],  c = eps[(samples - 1) n ..]      (eps.chunk(samples)[-2:])
 *   e = u + guidance * (c - u)
 *   s = *step_dev;  (a, r, k, d) = coef_dev[4 s .. 4 s + 3];  out <- k * ((x - a * e) * r) + d * e
 * with a = sigma, r = 1 / mu, k = mu_prev, d = sigma_prev (the rows ops.ddim_table builds).  A step outside
 * [0, n_steps) writes nothing.
 *   x_dev [n] fp16, the chunk's latents; eps_dev [samples, n] fp16, the UNet output of the chunk, samples 2
 *   ([uncond | cond]) or 3 (PnP's [source | uncond | cond]); out_dev [n] fp16, either x_dev itself or a buffer that
 *   overlaps neither x nor eps (VTM_E_SHAPE); any n >= 1; all three 2-byte aligned (VTM_E_SHAPE); coef_dev
 *   [n_steps, 4] fp32, 16-byte aligned; step_dev int32, 4-byte aligned.  NULL pointers: VTM_E_NULL.
 * Rounding is torch's, op for op: the guidance sub, mul and add each round to fp16, with `guidance` the fp32 value of
 * the caller's python float (the opmath scalar of torch's half mul); then KI's five roundings.  NaN and inf propagate
 * as through those torch ops.  16-byte vectors wherever x, u, c and out share their offset from a 16-byte boundary.
 * No allocation, no synchronisation: capturable in a CUDA graph, where one capture serves every step.
 */
int vtm_cfg_ddim_update_f16(const void* x_dev, const void* eps_dev, int64_t n, int32_t samples, float guidance,
                            const float* coef_dev, const int32_t* step_dev, int32_t n_steps, void* out_dev,
                            void* stream);

/*
 * KG1 / KG2 / NchwEpi — the entry and exit of diffusers' Transformer2DModel.forward, the module that owns every
 * BasicTransformerBlock of the UNet and works on NCHW activations (third-party code, not part of the reference; its
 * arithmetic is torch's):
 *   residual = x;  x = GroupNorm(groups, C)(x);  x = proj_in(x);  x -> [n, HW, C] tokens;  blocks;  x -> NCHW;
 *   x = proj_out(x);  return x + residual                (proj_in / proj_out: 1x1 Conv2d, or Linear on the token side)
 * x_dev is a contiguous NCHW fp16 tensor [n, C, HW], 2-byte aligned (16-byte aligned and HW % 8 == 0 for the vector
 * paths), C % groups == 0 (VTM_E_SHAPE).
 *
 * vtm_group_norm_stats_f16: stats_dev [n, groups, 2] fp32 = (mean, rstd) of every (sample, group), a contiguous run of
 *   (C / groups) * HW halfs; rstd = 1 / sqrt(var + eps) with the biased variance; fp32 throughout, combined pairwise
 *   (Chan et al.) so that a large mean does not cancel.  The partial sums start at x's first 16-byte boundary, so their
 *   rounding depends on x's offset from one: calls with the same offset agree bit for bit.  stats_dev 8-byte aligned,
 *   eps >= 0.  Workspace:
 *   vtm_group_norm_stats_workspace_bytes(n, C, HW, groups) (0 unless long runs are split over CTAs; VTM_E_WS).
 * vtm_group_norm_tokens_f16: y_dev [n, HW, C] fp16 token-major, 16-byte aligned, C % 8 == 0,
 *   y[i, p, c] = fp16(fma((float(x[i, c, p]) - mean) * rstd, gamma[c], beta[c])) with fp32 round-to-nearest steps;
 *   gamma_dev / beta_dev [C] fp16, NULL = 1 / 0.  n <= 65535.
 * vtm_linear_nchw_residual_f16: D[i, o, p] = fp16(fp16(sum_k A[i HW + p, k] W[o, k] + bias[o]) + R[i, o, p]),
 *   a_dev [n * HW, K] token-major rows, w_dev [N, K], bias_dev [N] or NULL, resid_dev [n, N, HW] or NULL, d_dev
 *   [n, N, HW]; K % 8 == 0, N % 8 == 0.  The mainloop, the bias and the two roundings are vtm_linear_residual_f16's:
 *   the result equals that entry's followed by a transpose, bit for bit.  d_dev may equal resid_dev.  d_dev and resid_dev
 *   need only be 2-byte aligned (16-byte aligned with HW % 8 == 0 takes the vector stores); the result is the same.
 */
size_t vtm_group_norm_stats_workspace_bytes(int32_t n, int32_t C, int32_t HW, int32_t groups);
int vtm_group_norm_stats_f16(const void* x_dev, int32_t n, int32_t C, int32_t HW, int32_t groups, float eps,
                             float* stats_dev, void* ws_dev, size_t ws_bytes, void* stream);
int vtm_group_norm_tokens_f16(const void* x_dev, const float* stats_dev, const void* gamma_dev, const void* beta_dev,
                              int32_t n, int32_t C, int32_t HW, int32_t groups, void* y_dev, void* stream);
int vtm_linear_nchw_residual_f16(const void* a_dev, const void* w_dev, const void* bias_dev, const void* resid_dev,
                                 int32_t n, int32_t HW, int32_t N, int32_t K, void* d_dev, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VIDTOME_B200_H_ */
