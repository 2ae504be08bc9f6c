/*
 * b200vit.h -- C ABI of libb200vit.so: hand-written sm_90a (H100) kernels for the ViT encoder forward path.
 *
 * The reference (lucidrains/vit-pytorch) is pure Python and has NO plugin / FFI interface;
 * its operator boundary for this path is the nn.Module surface.  Each entry point below therefore
 * names the reference *operator sequence* it replaces (file:line), and INTEGRATION.md shows the ctypes binding a
 * maintainer of the reference would add.
 *
 * Conventions
 *   - plain pointers and sizes only; no torch types.  All pointers are DEVICE pointers unless noted.
 *   - the caller owns every buffer (including workspaces); the library allocates nothing on the device.
 *   - all work is enqueued on `stream` (a cudaStream_t passed as void*) of the CURRENT device (the caller selects it,
 *     the library never calls cudaSetDevice); no internal synchronisation.  Entry points are re-entrant; per-device
 *     state (SM count, shared-memory attributes) is kept per device, tensor-map descriptors are cached per key.
 *   - return value 0 = success, negative = error; message via b200vit_last_error() (thread local).
 *   - bf16 = __nv_bfloat16 storage; accumulation, LayerNorm statistics, softmax and the residual stream are fp32.
 */
#ifndef B200VIT_H_
#define B200VIT_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200VIT_OK 0
#define B200VIT_ERR_INVALID -1  /* bad argument (shape, alignment, null pointer) */
#define B200VIT_ERR_CUDA -2     /* a CUDA runtime / driver call failed */
#define B200VIT_ERR_DEVICE -3   /* not an sm_90 device */

/* GEMM epilogue flags (b200vit_gemm_bf16) */
#define B200VIT_EPI_BIAS 1      /* + bias[n] (fp32) */
#define B200VIT_EPI_GELU 2      /* exact-erf GELU (nn.GELU default, vit.py:21) */
#define B200VIT_EPI_RESIDUAL 4  /* + resid[m, n] (fp32); resid may alias out_f32 (in-place residual stream) */
#define B200VIT_EPI_LNFOLD 8    /* A is the un-normalised bf16 row, W carries gamma: y = rstd_m*(acc - mu_m*s_n) + bias_n */
#define B200VIT_EPI_STATS 16    /* write per-row partial (sum, sum^2) of the bf16-rounded result into stats_out */
#define B200VIT_EPI_HEADLN 64   /* b200vit_gemm_headnorm_bf16: per-head LayerNorm (no bias) instead of the RMS norm */

const char* b200vit_last_error(void);
int b200vit_version(void);
/* number of kernels this library has launched in the calling process (all threads) since load / last reset */
int64_t b200vit_launch_count(void);
void b200vit_reset_launch_count(void);
/* 0 when device `dev` is sm_90 and the driver entry points the library needs resolve; negative otherwise */
int b200vit_device_ok(int dev);

/*
 * out[M, N] = epilogue( A[M, K] (bf16, row stride lda) x W[N, K]^T (bf16, row stride ldw) ), fp32 accumulate.
 * TMA-fed wgmma GEMM, persistent, warp specialised (one producer and two consumer warpgroups).  Replaces every nn.Linear on the path:
 *   vit.py:20,23 (FeedForward), vit.py:44,47 (to_qkv / to_out), vit.py:102 (patch projection), vit.py:116 (mlp_head);
 *   simple_vit.py:30,32,47,48,93,108.
 * out_bf16 and/or out_f32 (either may be NULL, not both), row stride ldo (elements).
 * EPI_LNFOLD: ln_sums[M][ln_parts][2] = per-row PARTIAL (sum, sum of squares) of A (added up in index order, so the
 *             result is deterministic), ln_dim = K, col_s[N] = sum_k W[n,k] (fp32).
 * EPI_STATS:  stats_out[M][P][2], P = b200vit_stats_parts(N): every slot is written exactly once (no atomics).
 * Requirements: A, W 16-byte aligned, lda, ldw multiples of 8, K multiple of 8.
 */
int b200vit_gemm_bf16(const void* A, int64_t lda, const void* W, int64_t ldw, void* out_bf16, float* out_f32,
                      int64_t ldo, const float* bias, const float* resid, const float* ln_sums, int ln_parts,
                      float ln_eps, const float* col_s, float* stats_out, int M, int N, int K, int flags,
                      void* stream);
/* number of per-row partial statistics an EPI_STATS GEMM with N output columns writes */
int b200vit_stats_parts(int N);

/*
 * LayerNorm over the last dim of an fp32 [M, D] matrix (row stride ldx) -> bf16 and/or fp32 outputs.
 * Replaces nn.LayerNorm(dim) at vit.py:19,39,69,103 / simple_vit.py:29,42,67,94 (eps 1e-5, biased variance).
 * gamma/beta fp32 [D] (beta may be NULL: NaViT's bias-free LayerNorm, na_vit.py:82-89).
 * If row_index != NULL, output row i is computed from input row row_index[i]  (cls pooling: vit.py:135).
 */
int b200vit_layernorm(const float* x, int64_t ldx, const float* gamma, const float* beta, void* out_bf16,
                      float* out_f32, int64_t ldo, const int32_t* row_index, int M, int D, float eps, void* stream);

/*
 * Patchify + LayerNorm(patch_dim): img[B, C, H, W] (bf16, NCHW contiguous) -> A[B*gh*gw, ldo] bf16 with
 *   A[b*(gh*gw) + h*gw + w, (p1*pw + p2)*C + c] = LN_over_patch(img[b, c, h*ph + p1, w*pw + p2]) * gamma + beta.
 * Replaces Rearrange('b c (h p1) (w p2) -> b (h w) (p1 p2 c)') + nn.LayerNorm(patch_dim), vit.py:100-101 /
 * simple_vit.py:91-92.  Columns [patch_dim, ldo) are zero filled (K padding for the GEMM).
 */
int b200vit_patchify_ln(const void* img, const float* gamma, const float* beta, void* out_bf16, int64_t ldo, int B,
                        int C, int H, int W, int ph, int pw, float eps, void* stream);

/*
 * Token assembly after the patch projection: y[B*n, D] (fp32, patch GEMM output incl. bias) ->
 *   x[b, t, :] = LN_D(y[b, t - ncls, :]) * gamma + beta + pos[t, :]   for t >= ncls
 *   x[b, 0, :] = cls[:] + pos[0, :]                                    if ncls == 1
 *   x[b, ncls + n + r, :] = tail[r, :]                                 for r < ntail (register tokens, no pos;
 *                                                                       simple_vit_with_register_tokens.py:124-126)
 * written as the fp32 residual stream x[B*(ncls+n+ntail), D].  Optional (may be NULL): xb_bf16 = bf16 copy of x and
 * stats[M][2] = per-row (sum, sum of squares) of that copy -- the inputs of the first LN-folded GEMM.
 * Replaces nn.LayerNorm(dim) vit.py:103, cls concat vit.py:122-123, pos add vit.py:125-127 (simple_vit.py:94,114).
 */
int b200vit_embed_tokens(const float* y, const float* gamma, const float* beta, const float* cls, const float* pos,
                         const float* tail, float* x, void* xb_bf16, float* stats, int B, int n, int ncls, int ntail,
                         int D, float eps, void* stream);

/*
 * im2col-free patch embedding for 16 x 16 patches (vit.py:100-102 without materialising the Rearrange or the
 * LayerNorm): y[B*n, D] fp32 = LN(patch pixels; gamma, beta) W^T + b, with the A operand of the wgmma GEMM loaded
 * straight out of the NCHW bf16 image by a 5-D TMA tensor map (pixel | pixel row | patch column | patch row |
 * image x channel), the LayerNorm folded into the epilogue.
 *   b200vit_patch_stats: stats[B*n][2] = (sum, sum of squares) of each patch's C*256 pixels.
 *   b200vit_patch_embed_tma: w_perm[D][C*256] bf16 = gamma (.) W with its columns permuted from the reference's
 *     (p1 p2 c) order to (c p1 p2); bias[D] = W beta + b; col_s[D] = row sums of w_perm; ldo = row stride of out_f32.
 * H, W multiples of 16 (other patch sizes: b200vit_patchify_ln + b200vit_gemm_bf16).
 */
int b200vit_patch_stats(const void* img, float* stats, int B, int C, int H, int W, void* stream);
int b200vit_patch_embed_tma(const void* img, const void* w_perm, const float* bias, const float* col_s,
                            const float* patch_stats, float ln_eps, float* out_f32, int64_t ldo, int B, int C, int H,
                            int W, int D, void* stream);

/* x[M, D] fp32 -> xb bf16 copy + stats[M][2] = (sum, sum of squares) of the bf16-rounded rows: entry into the
 * LN-folded layer chain for token matrices handed to Transformer.forward directly (reference mae.py:74). */
int b200vit_rowstats_cast(const float* x, void* xb_bf16, float* stats, int M, int D, void* stream);

/*
 * Multi-head softmax attention straight out of the packed QKV buffer:
 *   qkv[B*N, 3*H*dh] bf16 (columns: [q | k | v], each head-major h*dh + d; vit.py:54-55)
 *   out[B*N, H*dh]   bf16 (merged heads, vit.py:63) = softmax(q k^T * scale) v          (vit.py:57-62)
 * N <= 512 (longer sequences: b200vit_attention_varlen).  128-row query tiles, keys streamed in blocks with an
 * online softmax in fp32; S = QK^T and O = PV on the tensor cores (bf16 operands, fp32 accumulation).
 * dh = 64, or 80 (canonical ViT-H/14).
 */
int b200vit_attention(const void* qkv, void* out, int B, int N, int H, int dh, float scale, void* stream);

/*
 * Variable-length attention over PACKED sequences (any length): tokens [cu_seqlens[s], cu_seqlens[s+1]) of
 * qkv[total_tokens, 3*H*dh] attend only among themselves; out[total_tokens, H*dh].  This is the block-diagonal
 * "same image" attention of NaViT (na_vit.py:335-337 mask + 161-166 SDPA) without padding or an O(L^2) mask, and the
 * long-sequence (N > 512) path of ViT.  dh = 64 or 80.  cu_seqlens_dev[num_seqs+1] and tile_prefix_dev[num_seqs+1] (number of 128-row
 * query tiles before sequence s; tile_prefix[num_seqs] == total_tiles) are DEVICE int32 arrays built by the caller.
 */
int b200vit_attention_varlen(const void* qkv, void* out, const int32_t* cu_seqlens_dev, const int32_t* tile_prefix_dev,
                             int num_seqs, int total_tokens, int total_tiles, int H, int dh, float scale,
                             void* stream);

/*
 * NaViT patch extraction over a LIST of images of different resolutions + LayerNorm(patch_dim) without bias, one launch:
 *   out[cu[s] + h*gw_s + w, (c*p + p1)*p + p2] = LN_patch(img_s[c, h*p + p1, w*p + p2]) * gamma      (na_vit.py:300,350)
 * img_ptrs_dev[S]: device array of the (contiguous bf16 [C, H_s, W_s]) images' addresses; dims_dev[S][2] = (H_s, W_s);
 * cu_seqlens_dev[S+1] token offsets; row_prefix_dev[S+1] = number of patch rows before image s.
 */
int b200vit_patchify_varlen_ln(const int64_t* img_ptrs_dev, const int32_t* dims_dev, const int32_t* cu_seqlens_dev,
                               const int32_t* row_prefix_dev, const float* gamma, void* out_bf16, int64_t ldo, int S,
                               int total_rows, int max_w, int C, int p, float eps, void* stream);

/*
 * NaViT per-head q/k RMSNorm, in place on the packed qkv[T, 3*H*dh] buffer (q and k slices only):
 *   v <- v / max(||v||, 1e-12) * sqrt(dh) * gamma[h, d]    (na_vit.py:93-101,149-150).  gamma_qk fp32 [2][H][dh].
 */
int b200vit_qk_rmsnorm(void* qkv, const float* gamma_qk, int T, int H, int dh, void* stream);

/*
 * Linear + per-head RMSNorm in one pass (NaViT to_q / to_kv followed by q_norm / k_norm, na_vit.py:145-150):
 *   out[M, N] bf16 = epilogue(A W^T)   with flags in {EPI_BIAS, EPI_LNFOLD} exactly as b200vit_gemm_bf16, then the first
 *   norm_heads heads (dh = 64 columns each, from column 0) of every row are replaced by
 *   v / max(||v||, 1e-12) * sqrt(dh) * head_gamma[h, d]   (norm computed on the bf16-rounded projection, like the
 *   reference's bf16 module): b200vit_gemm_bf16 followed by b200vit_rmsnorm_heads / b200vit_layernorm_heads.
 *   flags | EPI_HEADLN: the heads get nn.LayerNorm(dh, bias=False) instead -- (v - mean) * rsqrt(var + head_eps) *
 *   head_gamma[h, d] -- the q / k norm of the nested-tensor NaViT (na_vit_nested_tensor.py:61-62,101-102).
 */
int b200vit_gemm_headnorm_bf16(const void* A, int64_t lda, const void* W, int64_t ldw, void* out_bf16, int64_t ldo,
                               const float* bias, const float* ln_sums, int ln_parts, float ln_eps,
                               const float* col_s, const float* head_gamma, int norm_heads, int dh, float head_eps,
                               int M, int N, int K, int flags, void* stream);

/*
 * The same normalisation on any row-major bf16 buffer: the `nheads` consecutive dh-wide heads that start at column 0
 * of every row buf[t*ld ...] (the k half of a [k | v] buffer for the attention pooling, na_vit.py:143-150);
 * gamma fp32 [nheads][dh].  ld in elements, multiple of 8; buf 16-byte aligned.
 */
int b200vit_rmsnorm_heads(void* buf, int64_t ld, const float* gamma, int T, int nheads, int dh, void* stream);
/* ... and its LayerNorm (no bias) flavour: (v - mean) * rsqrt(var + eps) * gamma[h, d] over each dh-wide head. */
int b200vit_layernorm_heads(void* buf, int64_t ld, const float* gamma, int T, int nheads, int dh, float eps,
                            void* stream);

/*
 * NaViT token assembly on the packed [T, D] matrix (na_vit.py:228,350-359): x = LayerNorm(y; gamma, no bias)
 * + pos_h[row of the token in its image's patch grid] + pos_w[column]; optional bf16 copy xb and stats[T][2] =
 * (sum, sum of squares) of that copy (entry statistics of the LN-folded layer chain, as b200vit_embed_tokens).
 * cu_seqlens_dev[S+1]; dims_dev[S][2] = (H_s, W_s) in pixels (grid width = W_s / p).  D multiple of 4.
 * pos_h[pos_h_rows][D], pos_w[pos_w_rows][D]: every image's patch grid must fit the tables (the reference raises an
 * index error otherwise, na_vit.py:354-359; the caller checks, the kernel additionally clamps the row index).
 */
int b200vit_embed_varlen(const float* y, const float* gamma, const float* pos_h, const float* pos_w, int pos_h_rows,
                         int pos_w_rows, const int32_t* cu_seqlens_dev, const int32_t* dims_dev, float* x,
                         void* xb_bf16, float* stats, int T, int D, int S, int p, float eps, void* stream);

/*
 * NaViT attention pooling (na_vit.py:371-387): out[s, h*dh:(h+1)*dh] = softmax_j(qn_h . k_jh) v_jh over the tokens j of
 * sequence s; kv[T, 2*H*dh] bf16 (k normalised, then v), qn[H*dh] fp32, cu_seqlens_dev[S+1] device int32, scale 1.
 */
int b200vit_attn_pool(const void* kv, const float* qn, const int32_t* cu_seqlens_dev, void* out, int S, int H, int dh,
                      void* stream);

/* Mean over the first n_pool tokens of every image: x[B, N, D] fp32 -> out[B, D] fp32 (vit.py:135 pool == 'mean',
 * simple_vit.py:117: n_pool = N; simple_vit_with_register_tokens.py:130-132: the patch tokens only). */
int b200vit_mean_pool(const float* x, float* out, int B, int N, int D, int n_pool, void* stream);

/* fp32 -> bf16 cast of a contiguous buffer of n elements (n multiple of 8). */
int b200vit_cast_f32_bf16(const float* x, void* out_bf16, int64_t n, void* stream);

/*
 * All encoder layers in one call (vit.py:78-81 / simple_vit.py:74-77), LayerNorm-folded schedule: per layer
 *   b200vit_gemm_bf16 (LN fold; b200vit_gemm_headnorm_bf16 if qk_gamma) -> b200vit_attention (N <= 512, else
 *   b200vit_attention_varlen) -> b200vit_gemm_bf16 (+ residual, statistics) -> b200vit_gemm_bf16 (LN fold, GELU)
 *   -> b200vit_gemm_bf16 (+ residual, statistics).
 * The host-side loop below the language boundary: one call instead of 5 x depth (small batches are host bound).
 * Weights are the LN-folded forms the Python engine prepares (engine.py TransformerEngine.prepared):
 *   *_wg = gamma (.) W rounded to bf16, *_s[n] = sum_k wg[n, k] (fp32, from the rounded weights), *_t = W beta (+ bias).
 * x[B*N, D] fp32 is the residual stream, updated in place.  primed != 0: ws->xb (bf16 copy of x) and ws->stats_in
 * ([M][2] row (sum, sum of squares) of that copy) were written by b200vit_embed_tokens; else they are computed here.
 * ws->stats_a / stats_b: [M][b200vit_stats_parts(D)][2] fp32 scratch; ws->qkv [M, 3*heads*dh], ws->o [M, heads*dh],
 * ws->h [M, hidden] bf16 scratch.  cu_seqlens / tile_prefix / total_tiles: only for N > 512 (B sequences of N tokens).
 */
typedef struct b200vit_layer {
  const void* qkv_wg;      /* [3*heads*dh, D] bf16 */
  const float* qkv_t;      /* [3*heads*dh] */
  const float* qkv_s;      /* [3*heads*dh] */
  const float* qk_gamma;   /* NULL, or [2][heads][dh]: per-head q / k RMSNorm (simple_vit_with_qk_norm.py:60-67) */
  const void* out_w;       /* [D, heads*dh] bf16 */
  const float* out_b;      /* [D] or NULL */
  const void* fc1_wg;      /* [hidden, D] bf16 */
  const float* fc1_t;      /* [hidden] */
  const float* fc1_s;      /* [hidden] */
  const void* fc2_w;       /* [D, hidden] bf16 */
  const float* fc2_b;      /* [D] or NULL */
  float ln1_eps, ln2_eps;
} b200vit_layer;
typedef struct b200vit_encoder_ws {
  void *xb, *qkv, *o, *h;
  float *stats_in, *stats_a, *stats_b;
} b200vit_encoder_ws;
int b200vit_encoder_blocks(const b200vit_layer* layers, int depth, float* x, const b200vit_encoder_ws* ws, int B, int N,
                           int D, int heads, int dh, int hidden, float scale, int primed,
                           const int32_t* cu_seqlens_dev, const int32_t* tile_prefix_dev, int total_tiles,
                           void* stream);

/*
 * TEST HOOKS -- process-global switches for A/B tests and bring-up; NOT part of the re-entrant API above (a value set
 * here changes every later call of every thread).  Production code never calls them.
 *   key 1: b200vit_attention key block: 0 / 1 = 64 keys (default), 2 = 128 keys
 *   key 11: b200vit_attention_varlen: 0 = 64-key blocks (default), 1 = 128-key blocks, 2 = 64-key blocks with half of
 *           the softmax exponentials on the FMA pipe
 *   key 12: BLOCK_N of b200vit_gemm_bf16: 0 = auto (256 when N > 128, else 128), 1 = 128, 2 = 256
 *   key 13: b200vit_attention: 0 = all softmax exponentials on MUFU (default), 1 = half of them on the FMA pipe
 */
int b200vit_debug_set(int key, int value);

#ifdef __cplusplus
}
#endif
#endif /* B200VIT_H_ */
