/*
 * anyloc_b200.h -- C ABI of libanyloc_b200.so (sm_90a).
 *
 * The reference (AnyLoc) is pure Python and has no FFI; the boundary it exposes
 * for this hot path is the Python class API of /root/reference/utilities.py.
 * Each entry point below cites the reference interface whose arithmetic it
 * replaces; the Python mirror of that API (anyloc_b200/utilities.py) binds
 * these symbols with ctypes (see INTEGRATION.md).
 *
 * Conventions: every pointer is a DEVICE pointer unless the name ends in _host;
 * every call enqueues work on `stream` (a cudaStream_t passed as void*) and
 * returns without synchronising; return value 0 = ok, negative = error (text
 * from anyloc_last_error(), thread-local).  No global state; workspaces are
 * caller-owned (sizes from the *_workspace_bytes functions).  There is NO CPU
 * fallback: without a CUDA device the compute calls return ANYLOC_ERR_CUDA.
 */
#ifndef ANYLOC_B200_H
#define ANYLOC_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ANYLOC_OK 0
#define ANYLOC_ERR_ARG (-1)
#define ANYLOC_ERR_CUDA (-2)
#define ANYLOC_ERR_WORKSPACE (-3)
#define ANYLOC_ERR_UNSUPPORTED (-4)

/* dist_mode: VLAD(dist_mode=...) utilities.py:660 */
#define ANYLOC_DIST_COSINE 0
#define ANYLOC_DIST_EUCLIDEAN 1
/* metric: get_top_k_recall(method=...) utilities.py:439-444 */
#define ANYLOC_METRIC_IP 0
#define ANYLOC_METRIC_L2 1
/* facet: DinoV2ExtractFeatures(facet=...) utilities.py:245-252,274-281 */
#define ANYLOC_FACET_QUERY 0
#define ANYLOC_FACET_KEY 1
#define ANYLOC_FACET_VALUE 2
#define ANYLOC_FACET_TOKEN 3
/* ffn kinds of the DINOv2 family (upstream dinov2/hub/backbones.py) */
#define ANYLOC_FFN_MLP 0
#define ANYLOC_FFN_SWIGLU 1

/* GEMM epilogues (internal building blocks, exported for parity tests) */
#define ANYLOC_EPI_BIAS 0          /* out = acc + bias                                   */
#define ANYLOC_EPI_BIAS_SPLIT 1    /* v = acc + bias           -> (hi,lo) tf32 pair      */
#define ANYLOC_EPI_GELU_SPLIT 2    /* v = gelu_erf(acc + bias) -> (hi,lo)                */
#define ANYLOC_EPI_SWIGLU_SPLIT 3  /* cols (2j,2j+1)=(x1,x2); v=silu(x1)*x2 -> (hi,lo)[j] */
#define ANYLOC_EPI_LS_RESID 4      /* out = resid + gamma * (acc + bias)                 */
/* GEMM input / SPLIT-output pair formats: x is carried as (hi, lo) with hi + lo ~ x to ~22 bits */
#define ANYLOC_PAIR_TF32 0         /* two fp32 arrays: hi = rna_tf32(x), lo = x - hi (kind::tf32 tensor path)          */
#define ANYLOC_PAIR_F16 1          /* two fp16 arrays of s*x (s power of two): hi = fp16(s x), lo = fp16(s x - hi);
                                      kind::f16 tensor path (2x rate); activations use s = 8, the epilogue's alpha
                                      undoes s_A*s_B.  Values beyond the fp16 range (|s x| > 65504) overflow. */
#define ANYLOC_PAIR_BF16 2         /* NOT a pair and NOT fp32-equivalent: one bf16 array of bf16_rn(x) (8 significant
                                      bits, fp32's exponent range), no lo array (every *_lo pointer NULL), no scale
                                      (alpha 1); one bf16 MMA per product instead of three.  Tensor-core engine only
                                      (wgmma GEMM at every M, mma.sync attention): ANYLOC_GEMM_SIMT returns
                                      ANYLOC_ERR_UNSUPPORTED.  Accumulators, LayerNorm statistics, softmax, the
                                      residual stream and every feature output stay fp32. */
#define ANYLOC_PAIR_FP8 3          /* NOT a pair and NOT fp32-equivalent: single e4m3 GEMM inputs with power-of-two scales.
                                      A GEMM's A operand is e4m3 rows q = e4m3_rn(x / s_r) with one fp32 scale s_r per
                                      row (the "lo" array carries the [M] scales); its B operand (a weight matrix) is
                                      one e4m3 array e4m3_rn(w / s_w) with one scale s_w per matrix, which the GEMM's
                                      alpha carries.  s = 2^k, k the smallest integer with max|x| / s <= 448, k >= -126;
                                      s = 1 for an all-zero row (anyloc_fp8_scale).  One e4m3 MMA per product,
                                      promoted into the fp32 accumulator every 128 elements of K; SPLIT outputs, the
                                      attention and the patch embedding are single bf16 (ANYLOC_PAIR_BF16).
                                      Tensor-core engine only. */
#define ANYLOC_PAIR_F16X1 4        /* NOT a pair and NOT fp32-equivalent: the hi array of ANYLOC_PAIR_F16 alone.  One fp16
                                      array of s*x, bit for bit the hi that ANYLOC_PAIR_F16 writes for the same input:
                                      Veltkamp's split rounds s*x to nearest at 11 significant bits, then cvt.rn packs
                                      it into fp16 (ties and values in the fp16 subnormal range may differ from
                                      __float2half_rn(s*x)).  Activations use s = 8, weights the per-tensor power of
                                      two s_w of the fp16 pairs (the weights' hi of anyloc_split_f16); alpha =
                                      1/(8 s_w).  No lo array (every *_lo pointer NULL).  One fp16 MMA per product;
                                      2^-11 relative per operand, 8x finer than single bf16, with fp16's range: an
                                      |s x| > 65504 overflows to Inf.  Tensor-core engine only (wgmma GEMM at every
                                      M, wgmma attention).  Accumulators, LayerNorm statistics, softmax, the residual
                                      stream and every feature output stay fp32. */
#define ANYLOC_PAIR_BF16X3 5       /* bf16 pairs, NOT fp32-equivalent: two bf16 arrays, hi = bf16_rn(x) and
                                      lo = bf16_rn(x - hi) (x - hi is exact in fp32), about 16 significant bits with
                                      fp32's exponent range; no scale (alpha 1 for activations and weights alike).  Both
                                      lo arrays are mandatory: a NULL a_lo, b_lo, out_lo (SPLIT epilogues) or y_lo returns
                                      ANYLOC_ERR_ARG (without its lo an operand is ANYLOC_PAIR_BF16).  Three bf16 MMAs
                                      per product, hi.hi + lo.hi + hi.lo, accumulated in fp32 with the fp16 pairs'
                                      round-to-nearest chunks.  The SPLIT epilogues, LayerNorm, im2col, the qkv tap and
                                      the attention write bf16 pairs.  Tensor-core engine only (wgmma GEMM at every M,
                                      wgmma attention): ANYLOC_GEMM_SIMT returns ANYLOC_ERR_UNSUPPORTED.  Accumulators,
                                      LayerNorm statistics, softmax, the residual stream and every feature output stay
                                      fp32.  Values beyond bf16's largest finite value (~3.39e38) round to Inf. */
/* GEMM engines */
#define ANYLOC_GEMM_AUTO 0
#define ANYLOC_GEMM_SIMT 1         /* fp32 FFMA (validation / odd shapes)               */
#define ANYLOC_GEMM_TC3 2          /* tensor cores (wgmma / mma.sync), 3-term split (tf32 or f16 by pair format) */

const char* anyloc_last_error(void);
int anyloc_version(void);
/* >0: compute capability *10 of the current device (90 on H100); <0: no usable device */
int anyloc_device_info(int* sm_count, size_t* smem_optin_bytes);

/* ------------------------------------------------------------ instrumentation (bench.py)
 * anyloc_launch_count: kernels launched by this library since load (all threads).
 * Profiling (off by default; not thread-safe): when enabled every launch group records a cudaEvent
 * pair on its stream; anyloc_profile_read synchronises them and returns, per category
 * (0 gemm_tc, 1 gemm_simt, 2 attention, 3 layernorm, 4 vit_misc, 5 vlad, 6 topk), the summed
 * device milliseconds, the number of launch groups and the summed algorithmic work
 * (FLOPs for 0-2, bytes otherwise), then clears the records. */
#define ANYLOC_PROF_CATEGORIES 7
long long anyloc_launch_count(void);
int anyloc_profile_enable(int on);
int anyloc_profile_read(double* ms, long long* groups, double* work);

/* ------------------------------------------------------------------ VLAD
 * Replaces VLAD.generate / generate_multi (utilities.py:819-926) incl. the
 * residuals of generate_res_vec (:956-962) and fpk.KMeans.predict (:849):
 *   x^ = x / max(|x|,1e-12)                (norm_descs)
 *   label = argmax_k sim(x, c_k)            (cosine: x.c_k/(|c_k|+1e-8); euclid: 2x.c_k-|c_k|^2;
 *                                            lowest k wins exact ties)
 *   V_k = sum_{label=k} (x^ - c_k);  V_k /= max(|V_k|,1e-12) (intra_norm);  V /= max(|V|,1e-12)
 * feats [B,N,D] fp32 row-major, n_valid [B] (nullable; rows >= n_valid[b] ignored, ragged lists),
 * centers [K,D], vlad [B,K*D], labels [B,N] int32 (nullable; -1 for ignored rows).
 */
/* Alignment (each entry below refuses a pointer short of it with ANYLOC_ERR_ARG, before anything runs, even with
 * nothing to do): feats, centers, vlad, ws and a prepared blob 16-byte (float4 rows; feats and the workspace's centre
 * copies also feed the tensor-core assignment, whose TMA needs 16 bytes, so an accepted buffer never changes the
 * route); n_valid and labels 4-byte. */
size_t anyloc_vlad_workspace_bytes(int B, int N, int D, int K);
int anyloc_vlad_generate(const float* feats, const int32_t* n_valid, const float* centers,
                         int B, int N, int D, int K, int dist_mode, int norm_descs, int intra_norm,
                         float* vlad, int32_t* labels, void* ws, size_t ws_bytes, void* stream);
/* Prepared vocabulary: VLAD.generate / generate_multi are called once per image (batch) with the SAME c_centers
 * (utilities.py:216-217 of scripts/dino_v2_vlad.py fits once, then :233-237 generates for every image), so the
 * centre normalisation c/(|c|+1e-8) of fpk cos_sim, its tf32 copy and norms can be computed once.
 * anyloc_vlad_prepare fills a caller-owned device blob (anyloc_vlad_prepared_bytes); anyloc_vlad_generate_prepared
 * is anyloc_vlad_generate minus the per-call centre-prep launch, on every route.  It only reads the blob, so concurrent
 * calls may share one once anyloc_vlad_prepare has completed; the blob must be re-prepared whenever the centres (or dist_mode) change.  Results are
 * bitwise identical to anyloc_vlad_generate. */
/* Alignment: anyloc_vlad_prepare centers 4-byte, prepared 16-byte (what its readers need); _prepared as
 * anyloc_vlad_generate, prepared 16-byte. */
size_t anyloc_vlad_prepared_bytes(int D, int K);
int anyloc_vlad_prepare(const float* centers, int D, int K, int dist_mode, void* prepared, size_t prepared_bytes,
                        void* stream);
int anyloc_vlad_generate_prepared(const float* feats, const int32_t* n_valid, const float* centers, void* prepared,
                                  size_t prepared_bytes, int B, int N, int D, int K, int dist_mode, int norm_descs,
                                  int intra_norm, float* vlad, int32_t* labels, void* ws, size_t ws_bytes, void* stream);
/* Hard VLAD at any vocabulary size (the reference's VLAD takes any num_clusters, utilities.py:657-662, :819-926;
 * scripts/dino_v2_vlad_ablations.sh lists num_clusters up to 256).  anyloc_vlad_generate(_prepared) accumulates in
 * shared memory and refuses shapes outside it; anyloc_vlad_generate_route(B, N, D, K) names the accumulation a shape
 * takes there: ANYLOC_VLAD_ROUTE_ACC3 / _ACC2, or ANYLOC_VLAD_ROUTE_SORTED where it refuses.
 * anyloc_vlad_generate_sorted takes the arguments of anyloc_vlad_generate_prepared (same assignment, labels_out and
 * results' meaning) and accepts every shape with D % 4 == 0: the per-image label sort, task table and multi-task
 * partial sums live in the workspace (anyloc_vlad_sorted_workspace_bytes), and every sum is taken in the order of
 * ACC3, so where ACC3 runs both give bitwise equal descriptors and labels.  Each image's descriptor is independent of
 * the other images of the batch.  No floating-point atomics. */
/* Alignment of anyloc_vlad_generate_sorted: as anyloc_vlad_generate_prepared. */
#define ANYLOC_VLAD_ROUTE_ACC3 0
#define ANYLOC_VLAD_ROUTE_ACC2 1
#define ANYLOC_VLAD_ROUTE_SORTED 2
int anyloc_vlad_generate_route(int B, int N, int D, int K);
size_t anyloc_vlad_sorted_workspace_bytes(int B, int N, int D, int K);
int anyloc_vlad_generate_sorted(const float* feats, const int32_t* n_valid, const float* centers, void* prepared,
                                size_t prepared_bytes, int B, int N, int D, int K, int dist_mode, int norm_descs,
                                int intra_norm, float* vlad, int32_t* labels, void* ws, size_t ws_bytes, void* stream);
/* Soft assignment (vlad_mode="soft", utilities.py:862-887):
 *   a[q,k] = softmax_k(soft_temp * cos(x_q, c_k))      (F.cosine_similarity :870-875, norms clamped at 1e-8)
 *   V_k    = sum_q a[q,k] * sum_c (x^_q - c_c)          (the reference weights the residuals to ALL centres by
 *                                                        cluster k's probability, :881-884)
 *   then intra / global normalisation as above.  assign [B,N,K] (nullable) receives a; padded rows get 0. */
/* Alignment: feats and ws 16-byte (float4 rows of x and of the normalised centres); n_valid, centers, vlad and
 * assign 4-byte (the accumulation reads and writes one fp32 at a time). */
int anyloc_vlad_generate_soft(const float* feats, const int32_t* n_valid, const float* centers,
                              int B, int N, int D, int K, float soft_temp, int norm_descs, int intra_norm,
                              float* vlad, float* assign, void* ws, size_t ws_bytes, void* stream);
/* Packed lists (VLAD.generate_multi of a list, whose items ext(list) returns as consecutive views of one buffer):
 * feats [R,D] fp32 rows, image b = rows [row0[b], row0[b] + len[b]) with row0 [B] int64 and len [B] int32 DEVICE
 * arrays, so one call serves any number of images without padding them to a common length.  Images may sit in any
 * order with rows between them that belong to none; len = 0 is allowed (a zero descriptor, as for an empty padded
 * image).  The call copies the table to the host (a synchronisation of `stream`) and returns ANYLOC_ERR_ARG, with
 * nothing launched, for len < 0, row0 < 0, row0 + len > R, two images sharing a row, B outside [0, 65535], R >= 2^31,
 * D not a multiple of 4, a null pointer, or feats / vlad not 16-byte, row0 not 8-byte or len not 4-byte aligned.
 * anyloc_vlad_generate_varlen takes the accumulation anyloc_vlad_generate_route(B, max len, D, K) names -- the route
 * of the padded batch [B, max len, D] -- and the descriptor of every image is bitwise the padded call's
 * (anyloc_vlad_generate_prepared / _sorted with n_valid = len); prepared is optional (NULL: centre prep per call).
 * labels [R] int32 (nullable): the padded call's label of each image row, -1 for rows of no image.  The soft form's
 * assign [R,K] (nullable) likewise: each image row's probabilities, 0 for rows of no image.  Workspaces:
 * anyloc_vlad_varlen_workspace_bytes(R, B, max len, D, K) and anyloc_vlad_soft_varlen_workspace_bytes(R, B, D, K). */
/* Alignment: the padded entries' (anyloc_vlad_generate_prepared / anyloc_vlad_generate_soft) plus row0 8-byte, len
 * 4-byte; the soft form's vlad stays 16-byte. */
size_t anyloc_vlad_varlen_workspace_bytes(int64_t R, int B, int max_len, int D, int K);
int anyloc_vlad_generate_varlen(const float* feats, int64_t R, const int64_t* row0, const int32_t* len, int B,
                                const float* centers, void* prepared, size_t prepared_bytes, int D, int K, int dist_mode,
                                int norm_descs, int intra_norm, float* vlad, int32_t* labels, void* ws, size_t ws_bytes,
                                void* stream);
size_t anyloc_vlad_soft_varlen_workspace_bytes(int64_t R, int B, int D, int K);
int anyloc_vlad_generate_soft_varlen(const float* feats, int64_t R, const int64_t* row0, const int32_t* len, int B,
                                     const float* centers, int D, int K, float soft_temp, int norm_descs,
                                     int intra_norm, float* vlad, float* assign, void* ws, size_t ws_bytes,
                                     void* stream);
/* Residual tensor of VLAD.generate_res_vec (utilities.py:928-972): out[q,k,:] = x^_q - c_k for ALL (patch, centre)
 * pairs, [N,K,D] fp32 (x^ = F.normalize(x) when norm_descs).  The reference builds every descriptor from this tensor
 * and caches it per image (`<cache_id>_r.pt`); here it is only materialised when a caller asks for it. */
/* Alignment: feats, centers and out 16-byte (float4). */
int anyloc_vlad_residuals(const float* feats, const float* centers, int N, int D, int K, int norm_descs,
                          float* out, void* stream);
/* Descriptor of ONE image from a residual tensor [N,K,D] plus either the hard labels [N] int32 (utilities.py:853-861)
 * or the soft assignment [N,K] (:879-887) -- the reference's cache path (`_r.pt` + `_l.pt` / `_s.pt`, :843-852,
 * :864-878), which needs no features.  Pass exactly one of labels / assign.  vlad [K*D]. */
/* Alignment: every pointer 4-byte (scalar kernels). */
size_t anyloc_vlad_from_residuals_workspace_bytes(int D, int K);
int anyloc_vlad_from_residuals(const float* resid, const int32_t* labels, const float* assign, int N, int D, int K,
                               int intra_norm, float* vlad, void* ws, size_t ws_bytes, void* stream);
/* labels only (fpk.KMeans.predict, utilities.py:849; also one Lloyd assignment step of VLAD.fit :786) */
/* Alignment: feats and ws 16-byte (as anyloc_vlad_generate), centers and labels 4-byte (the centre prep reads fp32). */
int anyloc_vlad_assign(const float* feats, const float* centers, int R, int D, int K, int dist_mode,
                       int32_t* labels, void* ws, size_t ws_bytes, void* stream);
/* one Lloyd centroid update of fpk.KMeans.fit (utilities.py:786): new_c[k] = mean of members
 * (0 for empty clusters); err_out[0] = sum((new_c - old_c)^2).  Deterministic (per-chunk partial sums added in a
 * fixed order, no floating-point atomics).  Workspace: anyloc_kmeans_workspace_bytes(R, D, K). */
/* Alignment of every k-means entry (update, _tiled, the rounds, _multi's labels[v] and ws[v], finalize): every pointer
 * 4-byte; the kernels read and write one fp32 / int32 at a time. */
size_t anyloc_kmeans_workspace_bytes(int R, int D, int K);
int anyloc_kmeans_update(const float* x, const int32_t* labels, const float* old_centers, int R, int D,
                         int K, float* new_centers, float* err_out, void* ws, size_t ws_bytes,
                         void* stream);
/* The same update in rounds, for rows that do not all fit on the device at once (VLAD.fit on host descriptors,
 * utilities.py:749-791; fpk's Lloyd loop restated in oracle/fpk_restated.py).  anyloc_kmeans_update splits R rows
 * into `chunks` contiguous chunks of `rows_per` rows (the last may be shorter) and sums each chunk sequentially;
 * anyloc_kmeans_partition returns that partition (it depends on R, D and the device's SM count).
 * anyloc_kmeans_accumulate_round takes one round: x [round_rows, D] and its labels hold, chunk after chunk, the next
 * `piece_rows` rows of every chunk (the last chunk's piece is round_rows - (chunks-1)*piece_rows rows, possibly 0).
 * resume=0 starts the per-chunk sums from zero, resume=1 continues those in the workspace.  After the last round,
 * anyloc_kmeans_finalize writes new_centers and err_out as anyloc_kmeans_update would: feeding each chunk's rows in
 * order, over any number of rounds, gives bit-identical centres.  R is the whole fit's row count in all three calls;
 * both compute calls use one workspace of anyloc_kmeans_round_workspace_bytes(R, D, K) bytes. */
int anyloc_kmeans_partition(int64_t R, int D, int* chunks, int64_t* rows_per);
size_t anyloc_kmeans_round_workspace_bytes(int64_t R, int D, int K);
int anyloc_kmeans_accumulate_round(const float* x, const int32_t* labels, int64_t R, int64_t round_rows,
                                   int64_t piece_rows, int D, int K, int resume, void* ws, size_t ws_bytes,
                                   void* stream);
int anyloc_kmeans_finalize(const float* old_centers, int64_t R, int D, int K, float* new_centers, float* err_out,
                           void* ws, size_t ws_bytes, void* stream);
/* The update and the round at any K (VLAD.fit with any num_clusters, utilities.py:749-791).  anyloc_kmeans_update and
 * anyloc_kmeans_accumulate_round keep K clusters' 128-column sums in 220 KB of shared memory, so they refuse
 * (K * 128 + K) * 4 > 220 KB (K >= 437).  The _tiled entries split the clusters into tiles of k_tile (0: the largest
 * that fits, 436); each tile reads its chunk's rows in order and adds those labelled inside it, so the partial sums,
 * centres, counts and err_out are bitwise those of the untiled entries wherever those run.  Same partition, workspace
 * (anyloc_kmeans_round_workspace_bytes), resume semantics and anyloc_kmeans_finalize. */
int anyloc_kmeans_accumulate_round_tiled(const float* x, const int32_t* labels, int64_t R, int64_t round_rows,
                                         int64_t piece_rows, int D, int K, int k_tile, int resume, void* ws,
                                         size_t ws_bytes, void* stream);
int anyloc_kmeans_update_tiled(const float* x, const int32_t* labels, const float* old_centers, int64_t R, int D,
                               int K, int k_tile, float* new_centers, float* err_out, void* ws, size_t ws_bytes,
                               void* stream);
/* Several vocabularies fitted on the same rows (fit_vocabularies): V vocabularies of K[v] centres each.
 * anyloc_vlad_assign_multi writes labels [V, R]; labels[v] equals anyloc_vlad_assign on vocabulary v alone, bit for
 * bit.  Each row is read once by one tf32 coarse GEMM over all sum K centres (rows in slices of at most 2^26 / sum K,
 * and at least 256) and once by the segmented rescoring.  A vocabulary for which anyloc_vlad_assign would take its
 * FFMA kernel (R < 256, D > 2048, a shape the GEMM refuses) takes it here too.  Workspace:
 * anyloc_vlad_assign_multi_workspace_bytes(R, D, V, K).
 * anyloc_kmeans_accumulate_round_multi is anyloc_kmeans_accumulate_round for each vocabulary v, with its labels[v],
 * K[v] and its own workspace ws[v] of anyloc_kmeans_round_workspace_bytes(R, D, K[v]) bytes: the partial sums are
 * bitwise the same, and anyloc_kmeans_finalize finishes each one.  It reads each row once per launch; consecutive
 * vocabularies share a launch while their sums and counts fit 220 KB of shared memory.  It refuses a K[v] that the
 * untiled round refuses (K >= 437). */
/* Alignment of anyloc_vlad_assign_multi: anyloc_vlad_assign's, each centers[v] 4-byte.  K, centers, labels (of
 * _multi) and ws_bytes are host arrays of pointers / sizes, read on the CPU. */
size_t anyloc_vlad_assign_multi_workspace_bytes(int64_t R, int D, int V, const int* K);
int anyloc_vlad_assign_multi(const float* feats, int64_t R, int D, int V, const float* const* centers, const int* K,
                             int dist_mode, int32_t* labels, void* ws, size_t ws_bytes, void* stream);
int anyloc_kmeans_accumulate_round_multi(const float* x, int V, const int32_t* const* labels, const int* K, int64_t R,
                                         int64_t round_rows, int64_t piece_rows, int D, int resume, void* const* ws,
                                         const size_t* ws_bytes, void* stream);
/* Several vocabularies' descriptors over the same features (generate_vocabularies): the per-row passes are shared,
 * each member's accumulation runs alone.
 * anyloc_vlad_label_multi writes labels [V, R] and inv_norm [R] = 1/max(|x|,1e-12) for R rows (a padded batch
 * [R/N, N, D] with n_valid, nullable, as in anyloc_vlad_generate; or packed rows).  labels[v] and inv_norm are
 * bitwise the labels and 1/|x| that vocabulary v's own generate call (anyloc_vlad_generate_prepared / _sorted /
 * _varlen) computes, labels -1 for rows n_valid leaves out.  inv_norm is unspecified on those rows (when the members
 * take different routes it may come from either; the accumulations never read it for a row labelled -1).  That call takes the tensor-core coarse pass plus exact rescoring
 * or the FFMA kernel by its own row count, which may break near-ties differently: route_rows[v] (host array, nullable
 * = R) is that count -- B * N of a padded call, B * max len of a packed one, whose R may be smaller.  Members on the
 * coarse route share one tf32 GEMM over all their centres per slice of rows and one rescoring read of each row.
 * prepared[v] (host array of anyloc_vlad_prepare blobs of prepared_bytes[v] bytes, nullable, entries nullable) stands
 * in for the centre prep as in the generate calls.  Workspace: anyloc_vlad_label_multi_workspace_bytes(R, D, V, K).
 * anyloc_vlad_soft_assign_multi writes each soft vocabulary's assignment assign[v] [R, K[v]] (K[v] <= 2048) at
 * temperature soft_temp[v] and inv_norm [R], bitwise anyloc_vlad_generate_soft(_varlen)'s assign and 1/|x|: one read of
 * each row and one dot product per (row, centre) for all members; rows n_valid leaves out get 0.  Workspace:
 * anyloc_vlad_soft_assign_multi_workspace_bytes(D, V, K).
 * anyloc_vlad_accumulate (padded [B,N,D]) and anyloc_vlad_accumulate_varlen (packed, table as above) run the
 * accumulation and normalisation of the generate calls from given per-row results: pass labels [rows] (hard; the
 * accumulation anyloc_vlad_generate_route(B, N, D, K) names, N the longest image for _varlen) OR assign [rows, K]
 * (soft; n_valid as in anyloc_vlad_generate_soft, ignored by the hard routes, which skip label -1), with inv_norm
 * [rows].  With the labels / assignment and inv_norm above the descriptors are bitwise the generate calls'.
 * Workspace of both: anyloc_vlad_accumulate_workspace_bytes(B, N, D, K, soft) (N = the longest len for _varlen; soft
 * != 0 sizes the soft accumulation, which needs only the sums of squares). */
/* Alignment: label_multi as anyloc_vlad_assign_multi plus n_valid and inv_norm 4-byte and each prepared[v] 16-byte;
 * soft_assign_multi feats and ws 16-byte, n_valid, inv_norm, each centers[v] and assign[v] 4-byte; the accumulates
 * feats, centers, vlad and ws 16-byte, n_valid, labels, assign, inv_norm and len 4-byte, row0 8-byte.  K, centers,
 * prepared, prepared_bytes, route_rows, soft_temp and the assign array are host arrays, read on the CPU. */
size_t anyloc_vlad_label_multi_workspace_bytes(int64_t R, int D, int V, const int* K);
int anyloc_vlad_label_multi(const float* feats, const int32_t* n_valid, int N, int64_t R, const int64_t* route_rows,
                            int D, int V, const float* const* centers, void* const* prepared,
                            const size_t* prepared_bytes, const int* K, int dist_mode, int32_t* labels, float* inv_norm,
                            void* ws, size_t ws_bytes, void* stream);
size_t anyloc_vlad_soft_assign_multi_workspace_bytes(int D, int V, const int* K);
int anyloc_vlad_soft_assign_multi(const float* feats, const int32_t* n_valid, int N, int64_t R, int D, int V,
                                  const float* const* centers, const int* K, const float* soft_temp,
                                  float* const* assign, float* inv_norm, void* ws, size_t ws_bytes, void* stream);
size_t anyloc_vlad_accumulate_workspace_bytes(int B, int N, int D, int K, int soft);
int anyloc_vlad_accumulate(const float* feats, const int32_t* n_valid, const int32_t* labels, const float* assign,
                           const float* inv_norm, const float* centers, int B, int N, int D, int K, int norm_descs,
                           int intra_norm, float* vlad, void* ws, size_t ws_bytes, void* stream);
int anyloc_vlad_accumulate_varlen(const float* feats, int64_t R, const int64_t* row0, const int32_t* len, int B,
                                  const int32_t* labels, const float* assign, const float* inv_norm,
                                  const float* centers, int D, int K, int norm_descs, int intra_norm, float* vlad,
                                  void* ws, size_t ws_bytes, void* stream);

/* ------------------------------------------------------------- retrieval
 * Replaces the faiss part of get_top_k_recall (utilities.py:435-450): optional row
 * normalisation (F.normalize), exact inner-product / squared-L2 scores, k best per query
 * sorted best-first, lowest database index first among equal scores.
 * db [n_db,Dv], qu [n_q,Dv] fp32; dist [n_q,k] fp32; idx [n_q,k] int64.
 */
/* Alignment of every retrieval entry (topk, index_*, index_split_*): db, qu, rows, ws, every index blob (index, dst,
 * src), a split index's host lo array and the stage 16-byte (float4 / uint4 rows and the score GEMM's TMA); dist
 * 4-byte; idx and the host counts 8-byte.  A blob or lo array is 16-byte in every entry that takes it. */
size_t anyloc_topk_workspace_bytes(int n_db, int n_q, int Dv, int k);
int anyloc_topk(const float* db, const float* qu, int n_db, int n_q, int Dv, int k, int metric,
                int normalize, float* dist, int64_t* idx, void* ws, size_t ws_bytes, void* stream);

/* Prepared database -- what `index.add(db)` leaves behind in faiss (utilities.py:449): the rows normalised (optional)
 * and stored as the (hi, lo) operand pairs the score GEMM consumes, plus |y|^2 per row (L2 metric).  Unit rows
 * (normalize != 0, Dv % 8 == 0) are kept as fp16 pairs of 4096*y (half the bytes, 2x tensor rate), other rows as tf32
 * pairs.  The blob is caller-owned (anyloc_index_bytes for `capacity` rows); rows can be added in chunks at any
 * row_offset (e.g. as descriptor batches arrive from the all-gather); a search over the first n_db rows is
 * anyloc_topk minus the per-call database pass.  `normalize` must be the same value in all calls on one blob.
 * anyloc_index_search: workspace from anyloc_index_search_workspace_bytes (query pairs + the [n_q, n_db] scores +
 * candidate lists).  Inner-product searches over an fp16-pair index run a hi-only (coarse) tensor-core pass with a
 * rigorous per-query error bound, re-score the candidates that could belong to the top-k exactly in fp32 and fall back
 * to the full 3-term product on the device when a candidate list overflows: same results, a third of the MMAs. */
size_t anyloc_index_bytes(int64_t capacity, int Dv, int normalize);
/* a fresh blob is initialised once before the first add; anyloc_index_copy moves the first n_rows rows into a larger
 * blob (growth) */
int anyloc_index_init(void* index, size_t index_bytes, int64_t capacity, int Dv, int normalize, void* stream);
int anyloc_index_copy(void* dst, size_t dst_bytes, int64_t dst_capacity, const void* src, size_t src_bytes,
                      int64_t src_capacity, int64_t n_rows, int Dv, int normalize, void* stream);
int anyloc_index_add(void* index, size_t index_bytes, int64_t capacity, int64_t row_offset, const float* rows,
                     int n_rows, int Dv, int normalize, void* stream);
size_t anyloc_index_search_workspace_bytes(int64_t n_db, int n_q, int Dv, int normalize);
int anyloc_index_search(const void* index, size_t index_bytes, int64_t capacity, int64_t n_db, const float* qu,
                        int n_q, int Dv, int k, int metric, int normalize, float* dist, int64_t* idx, void* ws,
                        size_t ws_bytes, void* stream);
/* Continuation form, for a database searched piece by piece (e.g. streamed from host memory): rows
 * [first, first + n_rows) of the blob are the global rows [row0, row0 + n_rows) of a database of n_total rows.  Their
 * k best are merged, in place and on the device, into the running list dist / idx [n_q, k] (global indices; score
 * descending, lowest index first).  A fresh list is -1 / -inf (IP) or -1 / +inf (L2) everywhere.  The route (coarse or
 * exact, see above) is chosen from n_total, not n_rows, and each route's score of a (query, row) pair does not depend
 * on where the row sits, so pieces fed in row order give what anyloc_index_search over the whole database gives --
 * except where the coarse route's 3-term fallback fires (it answers per piece).  k <= 4096.  Workspace:
 * anyloc_index_search_workspace_bytes(n_rows, n_q, Dv, normalize). */
int anyloc_index_search_continue(const void* index, size_t index_bytes, int64_t capacity, int64_t first,
                                 int64_t n_rows, int64_t row0, int64_t n_total, const float* qu, int n_q, int Dv, int k,
                                 int metric, int normalize, float* dist, int64_t* idx, void* ws, size_t ws_bytes,
                                 void* stream);
/* Split index: an fp16-pair inner-product index (normalize = 1, Dv % 8 == 0) whose lo halves stay in caller-owned
 * page-locked host memory, lo [capacity, Dv] fp16 (cudaHostAlloc or cudaHostRegister; the kernels reach it through its
 * unified address).
 * The device blob (anyloc_index_split_bytes for `capacity` rows) holds hi, |y|^2, dn and the header: about half of
 * anyloc_index_bytes.  Every stored value equals the resident index's, so searches return its (dist, idx) bit for bit.
 * anyloc_index_split_init / _copy / _add are anyloc_index_init / _copy / _add on this layout; _copy moves the device
 * part only (the caller copies lo rows [0, n_rows) to the new host array), _add writes lo into `lo` over the link. */
size_t anyloc_index_split_bytes(int64_t capacity, int Dv);
int anyloc_index_split_init(void* index, size_t index_bytes, int64_t capacity, int Dv, void* stream);
int anyloc_index_split_copy(void* dst, size_t dst_bytes, int64_t dst_capacity, const void* src, size_t src_bytes,
                            int64_t src_capacity, int64_t n_rows, int Dv, void* stream);
int anyloc_index_split_add(void* index, size_t index_bytes, int64_t capacity, void* lo, int64_t row_offset,
                           const float* rows, int n_rows, int Dv, void* stream);
/* The coarse route of a search over the first n_db rows, in two calls on one workspace
 * (anyloc_index_split_search_workspace_bytes).  anyloc_index_split_search: the hi-only pass and the candidate lists on
 * the device, the candidate rows de-duplicated and numbered in ascending row order, then ONE host synchronisation.
 * counts[0] = the unique candidate rows, counts[1] = the candidate rows summed over the queries.  counts[0] = -1: the
 * coarse route does not answer this batch (k > 64, n_db < 1024, n_q < 32, or a candidate list overflowed); answer it
 * by the exact route over pieces (anyloc_index_split_piece + anyloc_index_search_continue with n_total = n_db and
 * k > 64, whose first k columns are the resident answer: the same 3-term product and the same (score, index) order).
 * Otherwise anyloc_index_split_rescore writes the resident search's dist / idx [n_q, k].  With a stage of
 * anyloc_index_split_stage_bytes(counts[0], Dv) device bytes it gathers the unique rows' hi and lo (lo from host memory)
 * into the stage first and re-scores from there; with stage = NULL the re-scoring reads each candidate's lo row from
 * host memory directly, once per query that has it. */
size_t anyloc_index_split_search_workspace_bytes(int64_t n_db, int n_q, int Dv);
size_t anyloc_index_split_stage_bytes(int64_t rows, int Dv);
int anyloc_index_split_search(const void* index, size_t index_bytes, int64_t capacity, int64_t n_db, const float* qu,
                              int n_q, int Dv, int k, void* ws, size_t ws_bytes, int64_t* counts, void* stream);
int anyloc_index_split_rescore(const void* index, size_t index_bytes, int64_t capacity, const void* lo, int64_t n_db,
                               int n_q, int Dv, int k, void* ws, size_t ws_bytes, int64_t n_unique, void* stage,
                               size_t stage_bytes, float* dist, int64_t* idx, void* stream);
/* Rows [first, first + n_rows) of a split index as rows [0, n_rows) of an ordinary index blob (anyloc_index_bytes(
 * dst_capacity, Dv, 1)): hi, |y|^2 and dn copied on the device, lo copied from the host, the header (DN of the whole
 * index, a valid bound for the piece).  Asynchronous on `stream`; no init of `dst` is needed. */
int anyloc_index_split_piece(void* dst, size_t dst_bytes, int64_t dst_capacity, const void* index, size_t index_bytes,
                             int64_t capacity, const void* lo, int64_t first, int64_t n_rows, int Dv, void* stream);

/* ------------------------------------------------------------- collective
 * The one data-path collective of the pipeline (BASELINE config 4): all-gather of the [n_loc, Dv] fp32 descriptors of
 * every rank into [world * n_loc, Dv] (rank order), enqueued on `stream`.  `nccl_comm` is an ncclComm_t owned by the
 * caller (e.g. torch.distributed's NCCL backend); the library resolves ncclAllGather from the NCCL the process has
 * already loaded and returns ANYLOC_ERR_UNSUPPORTED when there is none.  The caller orders this call against its own
 * use of the communicator (one stream at a time per communicator). */
int anyloc_allgather_desc(void* nccl_comm, const float* local, float* all, size_t n_loc, int Dv, void* stream);

/* ------------------------------------------------------------------- ViT
 * Replaces DinoV2ExtractFeatures.__call__ (utilities.py:263-285) and the hub model's forward
 * it triggers (facebookresearch/dinov2 DinoVisionTransformer, see SURVEY.md App. A), with the
 * early exit at the hooked module (blocks 0..layer-1, then norm1+qkv-third or the whole block).
 */
typedef struct {
  int embed_dim;   /* 384 / 768 / 1024 / 1536 */
  int depth;       /* number of blocks whose weights are supplied */
  int num_heads;   /* head_dim must be 64 */
  int ffn_kind;    /* ANYLOC_FFN_* */
  int ffn_hidden;  /* 4*D (mlp) or 4096-style fused hidden (swiglu) */
  int patch;       /* 14 */
  int pair_dtype;  /* ANYLOC_PAIR_*: format of the weight pairs and of all GEMM-input activations (see below for
                      ANYLOC_PAIR_BF16) */
  int num_registers; /* R register tokens (dinov2_vit*14_reg: 4; 0 for the plain models) */
} AnylocVitCfg;

/* Per-block device pointers.  Matrices are [out,in] row-major like nn.Linear.weight, supplied as
 * tf32 (hi,lo) pairs with hi+lo == fp32 weight (anyloc_split_tf32).  For SwiGLU, w_in rows are
 * interleaved (row 2j = w12[j], row 2j+1 = w12[hidden+j]) and b_in likewise.
 * Alignment: every pointer of AnylocVitBlock 16-byte (the matrices, biases and LayerScale gammas are tensor-core GEMM
 * operands, the LayerNorm gains and biases float4 loads); in AnylocVitWeights patch_w_hi, patch_w_lo and patch_b
 * 16-byte, cls_token and register_tokens 4-byte; every AnylocVitTap out 16-byte. */
typedef struct {
  const float *ln1_w, *ln1_b;
  const void *qkv_w_hi, *qkv_w_lo; const float *qkv_b;     /* [3D,D], [3D] */
  const void *proj_w_hi, *proj_w_lo; const float *proj_b;  /* [D,D],  [D]  */
  const float *ls1;                                        /* [D] LayerScale gamma */
  const float *ln2_w, *ln2_b;
  const void *in_w_hi, *in_w_lo; const float *in_b;        /* fc1 [4D,D] or interleaved w12 [2H,D] */
  const void *out_w_hi, *out_w_lo; const float *out_b;     /* fc2 [D,4D] or w3 [D,H] */
  const float *ls2;
  /* accumulator scales 1/(s_act * s_weight) of the four GEMMs (1.0 for tf32 pairs) */
  float qkv_alpha, proj_alpha, in_alpha, out_alpha;
} AnylocVitBlock;

typedef struct {
  const void *patch_w_hi, *patch_w_lo;  /* [D, Kp] conv weight flattened (c,ky,kx), zero padded to Kp */
  const float *patch_b;                 /* [D] */
  const float *cls_token;               /* [D] */
  const AnylocVitBlock* blocks;         /* HOST array [depth] of device pointers */
  float patch_alpha;
  const float *register_tokens;         /* [R, D] (num_registers > 0), else unused */
} AnylocVitWeights;

/* Register tokens (upstream prepare_tokens with num_register_tokens = R): image b's token sequence is
 * [cls + pos[0], reg[0..R-1], patch[p] + pos[1+p]], T = 1 + R + N tokens; the registers get no positional embedding.
 * The output drops only the cls row (without use_cls), as DinoV2ExtractFeatures drops row 0 (utilities.py:273), so the
 * R register rows come first: [B, (1 +) R + N, D].  Every token count below (workspaces, the 32-bit token limit of the
 * _varlen calls) counts T per image.  R < 0, or R > 0 with a null register_tokens, returns ANYLOC_ERR_ARG (the
 * *_workspace_bytes functions return 0).  R = 0 is the plain model. */
/* Single bf16 (pair_dtype = ANYLOC_PAIR_BF16), the fast mode of every anyloc_vit_extract* call below: the weight
 * matrices are one bf16 array each (anyloc_split_bf16) with every *_w_lo NULL and every *_alpha 1; LayerNorm, im2col,
 * the qkv epilogue / tap and the attention write one bf16 array; the GEMMs and the attention run one bf16 MMA per
 * product.  The residual stream, LayerNorm statistics, softmax, every accumulator and every output stay fp32.  It is
 * not a parity mode: an output's error is that of the model run on bf16-rounded activations (about 2^-8 relative per
 * operand), not the 3-term formats' ~1e-6.  A non-NULL *_w_lo returns ANYLOC_ERR_ARG and gemm_engine =
 * ANYLOC_GEMM_SIMT ANYLOC_ERR_UNSUPPORTED, before anything is launched.  Every GEMM runs on the tensor cores whatever
 * M, so under ANYLOC_GEMM_AUTO too an image's rows are bit-identical across single, list (_varlen) and tap calls.
 * Workspace: with A(x) = x rounded up to 256 bytes, n_p patch rows, M token rows and H = ffn_hidden,
 *   A(2 n_p Kp) + A(4 n_p D) + A(4 M D) + A(2 M D) + A(6 M D) + A(2 M H) [+ A(12 M D) for the fp32 qkv rows of the
 *   tap calls, as below] + 4096 bytes. */
/* Single e4m3 (pair_dtype = ANYLOC_PAIR_FP8), a faster mode than single bf16: the block weight matrices (qkv, proj,
 * in, out) are e4m3 arrays e4m3_rn(w / s_w) (anyloc_quantize_fp8_tensor) with every *_w_lo NULL and *_alpha = s_w;
 * patch_w_hi is single bf16 (anyloc_split_bf16) with patch_w_lo NULL and patch_alpha 1.  LayerNorm writes e4m3 rows
 * and their scales in one pass; the qkv GEMM writes single bf16 for the bf16 attention (and the qkv tap); the
 * attention output and the FFN hidden layer are quantised to e4m3 rows (anyloc_quantize_fp8_rows) before the proj and
 * out GEMMs.  The patch embedding runs in single bf16.  The residual stream, LayerNorm statistics, softmax, every
 * accumulator and every output stay fp32.  Per-row activation scales keep an image's rows independent of the rows
 * around them, so single, list (_varlen) and tap calls are bit-identical as for single bf16.  A non-NULL *_w_lo returns
 * ANYLOC_ERR_ARG and gemm_engine = ANYLOC_GEMM_SIMT ANYLOC_ERR_UNSUPPORTED, before anything is launched.
 * Workspace: with A(x), n_p, M and H as above,
 *   A(2 n_p Kp) + A(4 n_p D) + A(4 M D) + A(M D) + A(4 M) + A(6 M D) + A(2 M H) + A(M H) + A(4 M) [+ A(12 M D) for
 *   the fp32 qkv rows of the tap calls] + 4096 bytes. */
/* Single fp16 (pair_dtype = ANYLOC_PAIR_F16X1), single bf16's speed at 2^-11 instead of 2^-8 per operand: the weight
 * matrices are the hi arrays of the fp16 pairs (anyloc_split_f16 with the pairs' per-tensor scale s_w, lo discarded),
 * every *_w_lo NULL and every *_alpha 1/(8 s_w); LayerNorm, im2col, the qkv epilogue / tap and the attention write one
 * fp16 array of 8 x; the GEMMs and the attention run one fp16 MMA per product.  What stays fp32 under single bf16 stays
 * fp32.  Not a parity mode; fp16's range applies (|8 x| > 65504 overflows to Inf, as for the fp16 pairs).  A non-NULL
 * *_w_lo returns ANYLOC_ERR_ARG and gemm_engine = ANYLOC_GEMM_SIMT ANYLOC_ERR_UNSUPPORTED, before anything is launched.
 * Every GEMM runs on the tensor cores whatever M, so single, list (_varlen) and tap calls are bit-identical.
 * Workspace: single bf16's formula (2-byte GEMM inputs, no lo buffers), with A(x), n_p, M and H as above:
 *   A(2 n_p Kp) + A(4 n_p D) + A(4 M D) + A(2 M D) + A(6 M D) + A(2 M H) [+ A(12 M D) for the fp32 qkv rows of the
 *   tap calls] + 4096 bytes. */
/* bf16 pairs (pair_dtype = ANYLOC_PAIR_BF16X3), fp32's exponent range at the fp16 pairs' speed: the weight matrices are
 * bf16 pairs (hi = anyloc_split_bf16 of w, lo = anyloc_split_bf16 of the fp32 remainder w - hi) with every *_w_lo
 * non-NULL and every *_alpha 1; LayerNorm, im2col, the qkv epilogue / tap and the attention write bf16 pairs; the GEMMs
 * and the attention run three bf16 MMAs per product.  What stays fp32 under single bf16 stays fp32.  Not a parity
 * mode: products keep about 16 significant bits, where the tf32 and fp16 pairs keep about 22; no scale, so nothing
 * overflows short of bf16's largest finite value.  A NULL *_w_lo returns ANYLOC_ERR_ARG and gemm_engine =
 * ANYLOC_GEMM_SIMT ANYLOC_ERR_UNSUPPORTED, before anything is launched.  Every GEMM runs on the tensor cores whatever
 * M, so single, list (_varlen) and tap calls are bit-identical.
 * Workspace: the 2-byte buffers of single bf16, each with its lo buffer, with A(x), n_p, M and H as above:
 *   2 A(2 n_p Kp) + A(4 n_p D) + A(4 M D) + 2 A(2 M D) + 2 A(6 M D) + 2 A(2 M H) [+ A(12 M D) for the fp32 qkv rows of
 *   the tap calls] + 4096 bytes. */
/* Alignment of every anyloc_vit_extract* call: ws and out (each taps_host[i].out) 16-byte (TMA and float4 access;
 * every buffer carved from ws inherits its alignment), img and pos_embed (each img[i] and pos_embed[i]) 4-byte, and the
 * weights as stated with AnylocVitBlock above, for every block 0..depth-1.  Anything else returns ANYLOC_ERR_ARG naming
 * the pointer, after the null, shape and tap checks and before the workspace size is checked or anything is launched. */
/* padded patch-embed reduction length (3*14*14=588 -> multiple of 32) */
int anyloc_vit_patch_k(int patch);
size_t anyloc_vit_workspace_bytes(const AnylocVitCfg* cfg, int B, int H, int W);
/* img [B,3,H,W] fp32 (H,W multiples of 14); pos_embed [1+g_h*g_w, D] already interpolated for this
 * grid (upstream interpolate_pos_encoding, with the model's own recipe); out [B, R + N (+1 if use_cls), D]. */
int anyloc_vit_extract(const AnylocVitCfg* cfg, const AnylocVitWeights* w_host, const float* img,
                       int B, int H, int W, const float* pos_embed, int layer, int facet,
                       int use_cls, int norm_descs, float* out, void* ws, size_t ws_bytes,
                       int gemm_engine, void* stream);

/* B images of DIFFERENT sizes in one forward pass.  Outside the benchmark datasets images keep their aspect ratio
 * (the reference demo, demo/anyloc_vlad_generate.py:160-185, shrinks the longest side to 1024 only when larger and
 * centre-crops to a multiple of 14), so two photos reach the ViT at different patch grids; padding them to one size
 * would change every softmax and the interpolated positional embedding.  Instead the token rows of all images are
 * packed one after another: the GEMMs and LayerNorms run once over all sum_i T_i rows, and the attention, im2col,
 * token assembly and facet slice read each image's geometry from a per-image table.
 *   img       HOST array of B device pointers; image i is [3, H_i, W_i] fp32
 *   hw        HOST int32 [B][2] = (H_i, W_i), positive multiples of the patch size
 *   pos_embed HOST array of B device pointers; pos_embed[i] = the table [1 + g_h,i * g_w,i, D] interpolated for image
 *             i's grid (images of the same grid may share one)
 *   out       packed [sum_i n_i, D] with n_i = R + g_h,i * g_w,i (+1 if use_cls); image i's rows start at sum_{j<i} n_j.
 * Each image's rows are bit-identical to anyloc_vit_extract on that image alone with the same GEMM engine (under
 * ANYLOC_GEMM_AUTO, a lone image of fewer than 32 tokens takes the SIMT GEMMs there, so compare those under TC3; the
 * single-bf16 format never does).
 * gemm_engine = ANYLOC_GEMM_SIMT returns ANYLOC_ERR_UNSUPPORTED: the packed attention is a tensor-core kernel.  The
 * call copies the geometry into kernel parameters; it neither synchronises with the host nor keeps any host pointer
 * it was given.  1 <= B <= ANYLOC_VIT_VARLEN_MAX_B. */
#define ANYLOC_VIT_VARLEN_MAX_B 128
size_t anyloc_vit_varlen_workspace_bytes(const AnylocVitCfg* cfg, int B, const int32_t* hw);
int anyloc_vit_extract_varlen(const AnylocVitCfg* cfg, const AnylocVitWeights* w_host, int B, const float* const* img,
                              const int32_t* hw, const float* const* pos_embed, int layer, int facet, int use_cls,
                              int norm_descs, float* out, void* ws, size_t ws_bytes, int gemm_engine, void* stream);

/* Several (layer, facet) features from ONE forward pass.  AnyLoc's results hinge on which layer and facet are read,
 * and its ablations sweep them: scripts/dino_v2_vlad_ablations.sh:16-25 runs layers {39..0} x facets,
 * scripts/dino_v2_vlad_viz.py:175-176 and dino_v2_vlad_viz_layers.py:370-376 build one DinoV2ExtractFeatures per layer
 * over the same images, scripts/dino_v2_sim_facets.py:145-151 reads all four facets of one layer.  The hooks of
 * utilities.py:245-252 define each facet: q/k/v of layer l are the thirds of blocks[l].attn.qkv(norm1(x)) (block l's
 * input), "token" is the output of blocks[l].  So blocks 0..L_max (the deepest tapped layer) run once each and every
 * tap keeps what that pass computes anyway.
 *   taps_host  HOST array of n_taps >= 1 distinct (layer, facet) pairs in any order, each with its own output: [B, R + N
 *              (+1 with use_cls), D] (anyloc_vit_extract_taps) or packed [sum_i n_i, D] (the _varlen form, layout as in
 *              anyloc_vit_extract_varlen).
 * Every output is bit-identical to anyloc_vit_extract / anyloc_vit_extract_varlen for that tap alone with the same
 * weights, images and GEMM engine; those two are the one-tap case of these calls.  An empty list, a layer outside
 * [0, depth), a bad facet, a repeated (layer, facet) or a null output returns ANYLOC_ERR_ARG, and a short workspace
 * ANYLOC_ERR_WORKSPACE, before anything is launched.  The call copies what it needs from taps_host, keeps no host
 * pointer and does not synchronise.  The workspace exceeds the one-tap size by M * 3D * 4 bytes (M = token rows) when
 * some layer's full fp32 qkv rows have to be kept: a layer with q/k/v taps below the deepest one, or a deepest layer
 * with a token tap and a q/k/v tap, or with two or three q/k/v taps. */
typedef struct {
  int layer;
  int facet;       /* ANYLOC_FACET_* */
  float* out;
} AnylocVitTap;
size_t anyloc_vit_taps_workspace_bytes(const AnylocVitCfg* cfg, int B, int H, int W, const AnylocVitTap* taps_host,
                                       int n_taps);
int anyloc_vit_extract_taps(const AnylocVitCfg* cfg, const AnylocVitWeights* w_host, const float* img, int B, int H,
                            int W, const float* pos_embed, const AnylocVitTap* taps_host, int n_taps, int use_cls,
                            int norm_descs, void* ws, size_t ws_bytes, int gemm_engine, void* stream);
size_t anyloc_vit_taps_varlen_workspace_bytes(const AnylocVitCfg* cfg, int B, const int32_t* hw,
                                              const AnylocVitTap* taps_host, int n_taps);
int anyloc_vit_extract_taps_varlen(const AnylocVitCfg* cfg, const AnylocVitWeights* w_host, int B,
                                   const float* const* img, const int32_t* hw, const float* const* pos_embed,
                                   const AnylocVitTap* taps_host, int n_taps, int use_cls, int norm_descs, void* ws,
                                   size_t ws_bytes, int gemm_engine, void* stream);

/* ------------------------------------------- building blocks (exported for parity tests)
 * C[M,N] = (A_hi+A_lo)[M,K] . (B_hi+B_lo)[N,K]^T with epilogue; *_lo nullable (treated as 0).
 * lda/ldb/ldo in elements.  out_lo/bias/gamma/resid per epilogue.
 * in_dtype = out_dtype = ANYLOC_PAIR_BF16: C = A . B^T of single bf16 operands (a_lo, b_lo, out_lo NULL, else
 * ANYLOC_ERR_ARG; bf16 in with another out_dtype, or the reverse, ANYLOC_ERR_ARG); the SPLIT epilogues write one bf16
 * array bf16_rn(v), BIAS / LS_RESID fp32 as usual.  Tensor-core engine only, at every M (SIMT: ANYLOC_ERR_UNSUPPORTED). */
/* in_dtype = out_dtype = ANYLOC_PAIR_F16X1: C = alpha A . B^T of single fp16 operands (a_lo, b_lo, out_lo NULL, else
 * ANYLOC_ERR_ARG; single fp16 in with another out_dtype, or the reverse, ANYLOC_ERR_ARG); the SPLIT epilogues write
 * one fp16 array, the hi of the fp16 pair of 8 v, BIAS / LS_RESID fp32.  Tensor-core engine only, at every M. */
/* in_dtype = out_dtype = ANYLOC_PAIR_BF16X3: C = alpha (A_hi.B_hi + A_lo.B_hi + A_hi.B_lo) of bf16-pair operands, a_lo
 * and b_lo mandatory (NULL: ANYLOC_ERR_ARG), out_lo mandatory for the SPLIT epilogues, which write the bf16 pair of v;
 * bf16 pairs in with another out_dtype, or the reverse, ANYLOC_ERR_ARG.  Tensor-core engine only, at every M. */
/* in_dtype = ANYLOC_PAIR_FP8, out_dtype = ANYLOC_PAIR_BF16: C = (s_r[m] alpha) (A . B^T) with A e4m3 [M, K] and its
 * fp32 row scales s_r in a_lo, B e4m3 (b_lo NULL) and alpha = s_w; out_lo NULL; the SPLIT epilogues write one bf16
 * array, BIAS / LS_RESID fp32.  K, lda and ldb multiples of 16.  Tensor-core engine only, at every M. */
int anyloc_gemm_nt(const void* a_hi, const void* a_lo, int lda, const void* b_hi, const void* b_lo,
                   int ldb, int M, int N, int K, int in_dtype, float alpha, int epilogue, const float* bias,
                   const float* gamma, const float* resid, void* out, void* out_lo, int ldo, int out_dtype,
                   int engine, void* stream);
/* which epilogue the calling thread's last tensor-core GEMM launch used: 1 = staged through shared memory and TMA
 * stores, 0 = stored from registers, -1 = none launched yet (a test observable; no effect on results) */
int anyloc_gemm_tc_last_staged(void);
int anyloc_split_tf32(const float* x, float* hi, float* lo, size_t n, void* stream);
int anyloc_split_f16(const float* x, void* hi, void* lo, size_t n, float scale, void* stream);
/* y = bf16_rn(x), the single-bf16 weight format */
int anyloc_split_bf16(const float* x, void* y, size_t n, void* stream);
/* y = LayerNorm(x) over rows of D (biased variance, eps inside the square root) with gain w and bias b, x [M, D] fp32.
 * out_dtype = ANYLOC_PAIR_TF32 / _F16: y_hi, y_lo [M, D] the pair of y (fp16 pairs: of 8 y);
 * out_dtype = ANYLOC_PAIR_BF16: y_hi = bf16_rn(LayerNorm(x)), y_lo NULL (else ANYLOC_ERR_ARG);
 * out_dtype = ANYLOC_PAIR_F16X1: y_hi = the hi array of the fp16 pair of 8 y, y_lo NULL (else ANYLOC_ERR_ARG);
 * out_dtype = ANYLOC_PAIR_BF16X3: y_hi, y_lo [M, D] the bf16 pair of y (y_lo NULL: ANYLOC_ERR_ARG);
 * out_dtype = ANYLOC_PAIR_FP8: y_hi = e4m3 rows of LayerNorm(x) [M, D], y_lo = their fp32 scales [M].
 * D a multiple of 4 in [4, 2048].  ANYLOC_ERR_ARG before anything is launched for a null pointer, M < 0, D outside that
 * range, x, w or b not 16-byte aligned, or y_hi / y_lo not aligned to 4 of their elements (fp8: y_hi and the scales
 * 4-byte aligned).  M = 0 launches nothing. */
int anyloc_layernorm_split(const float* x, const float* w, const float* b, int M, int D, float eps,
                           void* y_hi, void* y_lo, int out_dtype, void* stream);
/* The scale rule of ANYLOC_PAIR_FP8: the power of two s for a row or matrix whose largest magnitude is amax (host). */
float anyloc_fp8_scale(float amax);
/* bf16 rows x [M, K] -> e4m3 rows q [M, K] and their fp32 scales [M] (ANYLOC_PAIR_FP8's A operand).  K a multiple of 8;
 * x 16-byte, q 8-byte aligned.  Non-finite elements: a NaN becomes an e4m3 NaN and the row's scale is that of its
 * finite elements; a row that holds an Inf gets NaN bytes and a NaN scale, so the GEMM that consumes it writes a NaN
 * output row (e4m3 has no Inf, and saturating it to +-448 would leave the row finite and wrong).  The e4m3 LayerNorm
 * (anyloc_layernorm_split) does the same for a row whose output overflows fp32. */
int anyloc_quantize_fp8_rows(const void* x, int M, int K, void* q, float* scales, void* stream);
/* fp32 x [n] -> e4m3 q [n] = e4m3_rn(x / s) with one scale s, returned in *scale_host (a weight matrix of
 * ANYLOC_PAIR_FP8: its GEMM's alpha is s).  Synchronises the stream (the scale is chosen on the host); a NaN or Inf
 * in x returns ANYLOC_ERR_ARG. */
int anyloc_quantize_fp8_tensor(const float* x, void* q, size_t n, float* scale_host, void* stream);
/* softmax(q k^T / 8) v per head (head_dim 64).  qkv (hi,lo) pairs [B,T,3D] ([q|k|v] thirds); qkv_lo may
 * be NULL for the SIMT engine (plain fp32 input).  -> o (hi,lo) [B,T,D].  engine: ANYLOC_GEMM_*.
 * out_dtype = ANYLOC_PAIR_BF16: qkv_hi is single bf16 [B,T,3D] (what the qkv GEMM's bf16 split epilogue writes) and
 * o_hi single bf16 [B,T,D], qkv_lo and o_lo NULL (else ANYLOC_ERR_ARG); one bf16 MMA per product, P rounded once to
 * bf16, softmax in fp32; tensor cores only (ANYLOC_GEMM_SIMT: ANYLOC_ERR_UNSUPPORTED).
 * out_dtype = ANYLOC_PAIR_F16X1: the same with single fp16 qkv_hi of 8 x and o_hi of 8 o (the hi arrays of the fp16
 * pairs); 1/64 folded into the logit scale and P = 1024 p, as for the fp16 pairs, P rounded once.
 * out_dtype = ANYLOC_PAIR_BF16X3: qkv and o are bf16 pairs [B,T,3D] / [B,T,D], qkv_lo and o_lo mandatory (NULL:
 * ANYLOC_ERR_ARG); three bf16 MMAs per product, P split into a bf16 pair; tensor cores only, as for single bf16.
 * Alignment: o_hi and o_lo 8-byte (64-bit stores of the tensor-core epilogue), else ANYLOC_ERR_ARG before anything is
 * launched; a qkv that is not 16-byte aligned runs the SIMT kernel under ANYLOC_GEMM_AUTO (the single formats and
 * ANYLOC_GEMM_TC3: ANYLOC_ERR_UNSUPPORTED). */
int anyloc_attention(const float* qkv_hi, const float* qkv_lo, int B, int T, int D, int heads,
                     void* o_hi, void* o_lo, int out_dtype, int engine, void* stream);
/* The packed attention of the _varlen ViT calls, on n images of different lengths in one [rows, 3D] qkv buffer:
 * row0, len HOST int32 [n]; image i's q|k|v rows are [row0[i], row0[i] + len[i]) and its output rows the same rows of
 * o [rows, D].  Images may lie in any order with gaps between them; rows outside every image are neither used nor
 * written.  The operands are in the format fmt of the ViT's qkv epilogue, not converted: ANYLOC_PAIR_TF32 (tf32
 * pairs), ANYLOC_PAIR_F16 (fp16 pairs of 8*x, output pairs of 8*o), ANYLOC_PAIR_BF16X3 (bf16 pairs), ANYLOC_PAIR_BF16 or
 * ANYLOC_PAIR_F16X1 (qkv_lo, o_lo NULL).  The same
 * table (longest first) and launcher as the ViT; an image's rows are bit-identical to anyloc_attention on that image
 * alone (fp16 pairs: fed the tf32 pair of x) whatever the other images and the rows around it hold.
 * ANYLOC_ERR_ARG for a null pointer, n outside [1, ANYLOC_VIT_VARLEN_MAX_B], len[i] < 1, row0[i] < 0, overlapping
 * images, D != 64 heads, lo arrays with bf16 or without a pair format, a bad fmt, or o_hi / o_lo not 8-byte aligned;
 * ANYLOC_ERR_UNSUPPORTED for a qkv that is not 16-byte aligned.  Both return before anything is launched. */
int anyloc_attention_varlen(const void* qkv_hi, const void* qkv_lo, int n, const int32_t* row0, const int32_t* len,
                            int D, int heads, void* o_hi, void* o_lo, int fmt, void* stream);
/* y[r, :] = x[r, 0:D] / max(|x[r, 0:D]|, 1e-12) (F.normalize), x rows ld_in elements apart, y [rows, D] packed.
 * ANYLOC_ERR_ARG before anything is launched for a null pointer, rows < 0, D <= 0, D or ld_in not a multiple of 4,
 * ld_in < D, or x or y not 16-byte aligned.  rows = 0 launches nothing. */
int anyloc_l2_normalize_rows(const float* x, int64_t rows, int D, int64_t ld_in, float* y, void* stream);

/* ------------------------------------------------------------------ streamed PCA fit
 * The fit of reduce_pca (utilities.py:522-586, sklearn PCA(svd_solver="full")) for rows that do not fit on the device,
 * and the row passes of its randomized fit (svd_solver="randomized"):
 * the rows are fed in pieces and every sum lands in a caller-owned fp64 output that persists across calls.  x is fp32
 * [rows, cols], rows ld elements apart (ld >= cols); mu is fp64 [cols].  Each call sums in a fixed order, so the same
 * pieces give the same bits on every run.  Null pointers, negative sizes or ld < the row length return ANYLOC_ERR_ARG
 * before anything is launched; zero-sized calls launch nothing.
 *
 * anyloc_pca_colsum (utilities.py:522-586, the mean pass): sum[c] += sum_r x[r, c], in fp64.  Workspace
 * anyloc_pca_colsum_workspace_bytes(rows, cols); a short one returns ANYLOC_ERR_WORKSPACE. */
/* Alignment of the PCA entries: natural, for any ld -- x 4-byte; sum, ws, mu, u, out and a 8-byte. */
size_t anyloc_pca_colsum_workspace_bytes(int64_t rows, int cols);
int anyloc_pca_colsum(const float* x, int64_t ld, int64_t rows, int cols, double* sum, void* ws, size_t ws_bytes,
                      void* stream);
/* anyloc_pca_accumulate (utilities.py:522-586, the Gram / covariance matrix and vt): a centred A^T.B over the rows of
 * one piece on the FP64 tensor cores, each x element centred as (double)x - mu in registers.  out has ld_out >= its
 * columns; only its [out rows, out columns] elements are read and written.
 *   ANYLOC_PCA_COV  (n > d): out[cols, cols] += (x - mu)^T (x - mu), over a block of rows.  Lower-triangle 64x64 tiles
 *                   only; anyloc_pca_mirror completes the matrix.  u NULL, k unused.
 *   ANYLOC_PCA_GRAM (n <= d): out[rows, rows] += (x - mu)(x - mu)^T, over a slab of columns (x = those columns of all
 *                   rows, mu their means).  Lower-triangle tiles only, as above.  u NULL, k unused.
 *   ANYLOC_PCA_VT   out[k, cols] += u^T (x - mu), u fp64 [rows, k] (ld_u >= k; NULL only with k = 0), not centred: the Gram route's
 *                   vt = u[:, :k]^T Xc / s for one slab of columns (the caller divides by s), and the randomized fit's
 *                   W^T Xc over a block of rows.
 *   ANYLOC_PCA_SKETCH out[rows, k] += (x - mu) u, u fp64 [cols, k] (ld_u >= k; NULL only with k = 0), not centred: the
 *                   randomized fit's Xc W for a block of rows, contracting over the columns.  Every tile; rows <= 2^20. */
#define ANYLOC_PCA_COV 0
#define ANYLOC_PCA_GRAM 1
#define ANYLOC_PCA_VT 2
#define ANYLOC_PCA_SKETCH 3
int anyloc_pca_accumulate(int mode, const float* x, int64_t ld, int64_t rows, int cols, const double* mu,
                          const double* u, int64_t ld_u, int k, double* out, int64_t ld_out, void* stream);
/* anyloc_pca_mirror (utilities.py:522-586): a[i, j] = a[j, i] for j > i < m, after the last triangle accumulate, so
 * the matrix handed to the eigensolver is exactly symmetric. */
int anyloc_pca_mirror(double* a, int m, int64_t ld, void* stream);

/* ------------------------------------------------------------------ sibling aggregators
 * The pooling the reference's other DINOv2 scripts apply to the same patch features [B,N,D] -> [B,D]:
 *   ANYLOC_POOL_AVG  torch.mean(ret, dim=1)        scripts/dino_v2_gp.py:130-131
 *   ANYLOC_POOL_MAX  torch.max(ret, dim=1)[0]      scripts/dino_v2_gp.py:132-133
 *   ANYLOC_POOL_GEM  m = mean(x^p) (|x|^p with gem_use_abs); sign(m)|m|^(1/p)   scripts/dino_v2_gem.py:170-189
 * n_valid [B] nullable (ragged batches): image b pools its first min(N, n_valid[b]) rows and never reads the rest.  An
 * image with n_valid[b] <= 0 is empty and is written NaN in every mode (torch's mean of an empty set; max has no value
 * to give).  ANYLOC_ERR_ARG before anything is launched for a null pointer, B outside [0, 65535], N <= 0, D not a
 * positive multiple of 4, an unknown mode, gem_p = 0 with ANYLOC_POOL_GEM, or feats or out not 16-byte aligned (float4
 * access).  B = 0 launches nothing. */
#define ANYLOC_POOL_AVG 0
#define ANYLOC_POOL_MAX 1
#define ANYLOC_POOL_GEM 2
/* Alignment: feats and out 16-byte (float4), n_valid 4-byte. */
int anyloc_pool(const float* feats, const int32_t* n_valid, int B, int N, int D, int mode, float gem_p,
                int gem_use_abs, float* out, void* stream);
/* The same pooling of a packed list: feats [R,D], image b = rows [row0[b], row0[b] + len[b]) (row0 [B] int64, len [B]
 * int32, device arrays; the table rules and refusals of anyloc_vlad_generate_varlen, out 16-byte aligned in vlad's
 * place).  Each image's rows are read in pool's order, so out[b] is bitwise anyloc_pool's for the padded batch with
 * n_valid = len; len = 0 gives NaN.  No workspace.  Alignment: feats and out 16-byte, row0 8-byte, len 4-byte, checked
 * before B = 0 returns. */
int anyloc_pool_varlen(const float* feats, int64_t R, const int64_t* row0, const int32_t* len, int B, int D, int mode,
                       float gem_p, int gem_use_abs, float* out, void* stream);

/* ------------------------------------------------------------------ image pre-processing
 * Replaces `base_transform` (dvgl_benchmark/datasets_ws.py:20-23: T.ToTensor + T.Normalize) and the centre crop to a
 * multiple of the patch size (scripts/dino_v2_vlad.py:174-176) in one pass:
 *   out[b,c,y,x] = ((float)img[b,top+y,left+x,c] / 255 - mean[c]) / std[c]     (bit-identical to torchvision)
 * img [B,H,W,3] uint8 (device), mean3/std3 HOST arrays of 3 floats, out [B,3,Hc,Wc] fp32 (device).  out must be 4-byte
 * aligned, and 8-byte aligned when Wc is even (pairs of columns are stored as float2); ANYLOC_ERR_ARG otherwise, before
 * anything is launched. */
int anyloc_preprocess_u8(const uint8_t* img, int B, int H, int W, int top, int left, int Hc, int Wc,
                         const float* mean3, const float* std3, float* out, void* stream);
/* The same with the dataset loader's resize in between (dvgl_benchmark/datasets_ws.py:222-239
 * `T.functional.resize(base_transform(img), [480, 640])`; demo/anyloc_vlad_generate.py:165-177 bicubic down-scaling of
 * over-sized images): ToTensor + Normalize, ANTIALIASED resize to Hr x Wr (interpolation 0 = bilinear, 1 = bicubic --
 * torchvision's tensor defaults, i.e. torch interpolate(align_corners=False, antialias=True)), then the crop window
 * [top, top+Hc) x [left, left+Wc) of the resized image.  out [B,3,Hc,Wc], 4-byte aligned (else ANYLOC_ERR_ARG). */
int anyloc_preprocess_resize_u8(const uint8_t* img, int B, int H, int W, int Hr, int Wr, int interpolation, int top,
                                int left, int Hc, int Wc, const float* mean3, const float* std3, float* out,
                                void* stream);
/* A list of n differently sized photos, the two ways they reach AnyLoc: the demo's "your own images" path
 * (demo/anyloc_vlad_generate.py:160-185: each photo normalised, bicubic-resized to a 1024 long side with the aspect
 * ratio kept when larger, centre-cropped to multiples of 14, so every photo keeps its own size) and the dataset loader
 * (dvgl_benchmark/datasets_ws.py:222-239: every photo resized to 480x640 whatever its source size).
 * Image i: imgs[i] a DEVICE pointer to uint8 [H[i], W[i], 3]; with interpolation 0 (bilinear) or 1 (bicubic) it is
 * resized to Hr[i] x Wr[i] and the window [top[i], +Hc[i]) x [left[i], +Wc[i]) of the resized image is written, each
 * image bit-identical to anyloc_preprocess_resize_u8 on that image alone; with interpolation -1 there is no resize (Hr,
 * Wr may be NULL), the window is taken from the source image, and each image is bit-identical to anyloc_preprocess_u8.
 * Its output [3, Hc[i], Wc[i]] fp32 starts at out + out_offset[i] (floats).  imgs, H, W, Hr, Wr, top, left, Hc, Wc,
 * out_offset, mean3 and std3 are HOST arrays.  Up to ANYLOC_PREPROCESS_VARLEN_BATCH images per launch; a longer list
 * takes consecutive launches on the stream.  ANYLOC_ERR_ARG for a null pointer, an unknown interpolation, a crop
 * outside the (resized) image, a zero std, a negative offset, an out that is not 4-byte aligned, a horizontal
 * down-scaling beyond the 64-tap window or a launch over the grid limit -- all checked before the first launch, so a
 * refusal writes nothing.  Never synchronises
 * with the host.  n = 0 launches nothing. */
#define ANYLOC_PREPROCESS_VARLEN_BATCH 64
int anyloc_preprocess_u8_varlen(int n, const uint8_t* const* imgs, const int* H, const int* W, const int* Hr,
                                const int* Wr, int interpolation, const int* top, const int* left, const int* Hc,
                                const int* Wc, const float* mean3, const float* std3, float* out,
                                const int64_t* out_offset, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ANYLOC_B200_H */
