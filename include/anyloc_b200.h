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
size_t anyloc_vlad_prepared_bytes(int D, int K);
int anyloc_vlad_prepare(const float* centers, int D, int K, int dist_mode, void* prepared, size_t prepared_bytes,
                        void* stream);
int anyloc_vlad_generate_prepared(const float* feats, const int32_t* n_valid, const float* centers, void* prepared,
                                  size_t prepared_bytes, int B, int N, int D, int K, int dist_mode, int norm_descs,
                                  int intra_norm, float* vlad, int32_t* labels, void* ws, size_t ws_bytes, void* stream);
/* Soft assignment (vlad_mode="soft", utilities.py:862-887):
 *   a[q,k] = softmax_k(soft_temp * cos(x_q, c_k))      (F.cosine_similarity :870-875, norms clamped at 1e-8)
 *   V_k    = sum_q a[q,k] * sum_c (x^_q - c_c)          (the reference weights the residuals to ALL centres by
 *                                                        cluster k's probability, :881-884)
 *   then intra / global normalisation as above.  assign [B,N,K] (nullable) receives a; padded rows get 0. */
int anyloc_vlad_generate_soft(const float* feats, const int32_t* n_valid, const float* centers,
                              int B, int N, int D, int K, float soft_temp, int norm_descs, int intra_norm,
                              float* vlad, float* assign, void* ws, size_t ws_bytes, void* stream);
/* Residual tensor of VLAD.generate_res_vec (utilities.py:928-972): out[q,k,:] = x^_q - c_k for ALL (patch, centre)
 * pairs, [N,K,D] fp32 (x^ = F.normalize(x) when norm_descs).  The reference builds every descriptor from this tensor
 * and caches it per image (`<cache_id>_r.pt`); here it is only materialised when a caller asks for it. */
int anyloc_vlad_residuals(const float* feats, const float* centers, int N, int D, int K, int norm_descs,
                          float* out, void* stream);
/* Descriptor of ONE image from a residual tensor [N,K,D] plus either the hard labels [N] int32 (utilities.py:853-861)
 * or the soft assignment [N,K] (:879-887) -- the reference's cache path (`_r.pt` + `_l.pt` / `_s.pt`, :843-852,
 * :864-878), which needs no features.  Pass exactly one of labels / assign.  vlad [K*D]. */
size_t anyloc_vlad_from_residuals_workspace_bytes(int D, int K);
int anyloc_vlad_from_residuals(const float* resid, const int32_t* labels, const float* assign, int N, int D, int K,
                               int intra_norm, float* vlad, void* ws, size_t ws_bytes, void* stream);
/* labels only (fpk.KMeans.predict, utilities.py:849; also one Lloyd assignment step of VLAD.fit :786) */
int anyloc_vlad_assign(const float* feats, const float* centers, int R, int D, int K, int dist_mode,
                       int32_t* labels, void* ws, size_t ws_bytes, void* stream);
/* one Lloyd centroid update of fpk.KMeans.fit (utilities.py:786): new_c[k] = mean of members
 * (0 for empty clusters); err_out[0] = sum((new_c - old_c)^2).  Deterministic (per-chunk partial sums added in a
 * fixed order, no floating-point atomics).  Workspace: anyloc_kmeans_workspace_bytes(R, D, K). */
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

/* ------------------------------------------------------------- retrieval
 * Replaces the faiss part of get_top_k_recall (utilities.py:435-450): optional row
 * normalisation (F.normalize), exact inner-product / squared-L2 scores, k best per query
 * sorted best-first, lowest database index first among equal scores.
 * db [n_db,Dv], qu [n_q,Dv] fp32; dist [n_q,k] fp32; idx [n_q,k] int64.
 */
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
  int pair_dtype;  /* ANYLOC_PAIR_*: format of the weight pairs and of all GEMM-input activations */
  int num_registers; /* R register tokens (dinov2_vit*14_reg: 4; 0 for the plain models) */
} AnylocVitCfg;

/* Per-block device pointers.  Matrices are [out,in] row-major like nn.Linear.weight, supplied as
 * tf32 (hi,lo) pairs with hi+lo == fp32 weight (anyloc_split_tf32).  For SwiGLU, w_in rows are
 * interleaved (row 2j = w12[j], row 2j+1 = w12[hidden+j]) and b_in likewise. */
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
 * ANYLOC_GEMM_AUTO, a lone image of fewer than 32 tokens takes the SIMT GEMMs there, so compare those under TC3).
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
 * lda/ldb/ldo in elements.  out_lo/bias/gamma/resid per epilogue. */
int anyloc_gemm_nt(const void* a_hi, const void* a_lo, int lda, const void* b_hi, const void* b_lo,
                   int ldb, int M, int N, int K, int in_dtype, float alpha, int epilogue, const float* bias,
                   const float* gamma, const float* resid, void* out, void* out_lo, int ldo, int out_dtype,
                   int engine, void* stream);
/* which epilogue the calling thread's last tensor-core GEMM launch used: 1 = staged through shared memory and TMA
 * stores, 0 = stored from registers, -1 = none launched yet (a test observable; no effect on results) */
int anyloc_gemm_tc_last_staged(void);
int anyloc_split_tf32(const float* x, float* hi, float* lo, size_t n, void* stream);
int anyloc_split_f16(const float* x, void* hi, void* lo, size_t n, float scale, void* stream);
int anyloc_layernorm_split(const float* x, const float* w, const float* b, int M, int D, float eps,
                           void* y_hi, void* y_lo, int out_dtype, void* stream);
/* softmax(q k^T / 8) v per head (head_dim 64).  qkv (hi,lo) pairs [B,T,3D] ([q|k|v] thirds); qkv_lo may
 * be NULL for the SIMT engine (plain fp32 input).  -> o (hi,lo) [B,T,D].  engine: ANYLOC_GEMM_*. */
int anyloc_attention(const float* qkv_hi, const float* qkv_lo, int B, int T, int D, int heads,
                     void* o_hi, void* o_lo, int out_dtype, int engine, void* stream);
int anyloc_l2_normalize_rows(const float* x, int64_t rows, int D, int64_t ld_in, float* y, void* stream);

/* ------------------------------------------------------------------ sibling aggregators
 * The pooling the reference's other DINOv2 scripts apply to the same patch features [B,N,D] -> [B,D]:
 *   ANYLOC_POOL_AVG  torch.mean(ret, dim=1)        scripts/dino_v2_gp.py:130-131
 *   ANYLOC_POOL_MAX  torch.max(ret, dim=1)[0]      scripts/dino_v2_gp.py:132-133
 *   ANYLOC_POOL_GEM  m = mean(x^p) (|x|^p with gem_use_abs); sign(m)|m|^(1/p)   scripts/dino_v2_gem.py:170-189
 * n_valid [B] nullable (ragged batches). */
#define ANYLOC_POOL_AVG 0
#define ANYLOC_POOL_MAX 1
#define ANYLOC_POOL_GEM 2
int anyloc_pool(const float* feats, const int32_t* n_valid, int B, int N, int D, int mode, float gem_p,
                int gem_use_abs, float* out, void* stream);

/* ------------------------------------------------------------------ image pre-processing
 * Replaces `base_transform` (dvgl_benchmark/datasets_ws.py:20-23: T.ToTensor + T.Normalize) and the centre crop to a
 * multiple of the patch size (scripts/dino_v2_vlad.py:174-176) in one pass:
 *   out[b,c,y,x] = ((float)img[b,top+y,left+x,c] / 255 - mean[c]) / std[c]     (bit-identical to torchvision)
 * img [B,H,W,3] uint8 (device), mean3/std3 HOST arrays of 3 floats, out [B,3,Hc,Wc] fp32 (device). */
int anyloc_preprocess_u8(const uint8_t* img, int B, int H, int W, int top, int left, int Hc, int Wc,
                         const float* mean3, const float* std3, float* out, void* stream);
/* The same with the dataset loader's resize in between (dvgl_benchmark/datasets_ws.py:222-239
 * `T.functional.resize(base_transform(img), [480, 640])`; demo/anyloc_vlad_generate.py:165-177 bicubic down-scaling of
 * over-sized images): ToTensor + Normalize, ANTIALIASED resize to Hr x Wr (interpolation 0 = bilinear, 1 = bicubic --
 * torchvision's tensor defaults, i.e. torch interpolate(align_corners=False, antialias=True)), then the crop window
 * [top, top+Hc) x [left, left+Wc) of the resized image.  out [B,3,Hc,Wc]. */
int anyloc_preprocess_resize_u8(const uint8_t* img, int B, int H, int W, int Hr, int Wr, int interpolation, int top,
                                int left, int Hc, int Wc, const float* mean3, const float* std3, float* out,
                                void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ANYLOC_B200_H */
