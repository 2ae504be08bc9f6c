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
#define B200VIT_EPI_RESIDUAL 4  /* + resid[m, n] (fp32, row stride ldo, a multiple of 4); resid is either out_f32
                                   itself (in-place residual stream) or does not overlap it */
#define B200VIT_EPI_LNFOLD 8    /* A is the un-normalised bf16 row, W carries gamma: y = rstd_m*(acc - mu_m*s_n) + bias_n */
#define B200VIT_EPI_STATS 16    /* write per-row partial (sum, sum^2) of the bf16-rounded result into stats_out */
#define B200VIT_EPI_HARDSWISH 32  /* y * clamp(y + 3, 0, 6) / 6 after the bias, where GELU would be (nn.Hardswish,
                                     levit.py:32); not with B200VIT_EPI_GELU */
#define B200VIT_EPI_HEADLN 64   /* b200vit_gemm_headnorm_bf16: per-head LayerNorm (no bias) instead of the RMS norm */
#define B200VIT_EPI_SILU 128    /* y / (1 + exp(-y)) after the bias, where GELU would be (nn.SiLU, max_vit.py:55) */
#define B200VIT_EPI_SIGMOID 256 /* 1 / (1 + exp(-y)) after the bias, where GELU would be (nn.Sigmoid, max_vit.py:57);
                                   at most one of EPI_GELU, EPI_HARDSWISH, EPI_SILU and EPI_SIGMOID per call, and
                                   neither EPI_SILU nor EPI_SIGMOID with EPI_RESIDUAL */

/* attention flags (b200vit_attention_ex, b200vit_attention_varlen_ex, b200vit_encoder_blocks_ex) */
#define B200VIT_ATTN_MASK_SELF 1  /* key i of query i gets probability 0 (LSA, vit_for_small_dataset.py:53-57) */
/* b200vit_attention_posbias only (the entry points above reject it): exact-erf GELU on every fp32 output before it is
 * rounded to bf16 (LeViT's to_out, levit.py:60-61) */
#define B200VIT_ATTN_GELU_OUT 4
#define B200VIT_ATTN_POSBIAS_MAX_KEYS 4096  /* keys per image (F*F) of b200vit_attention_posbias */

/* what the convolutional tokenizer's kernels are built for (b200vit_conv_im2col_*, b200vit_relu_maxpool,
 * b200vit_seq_pool) */
#define B200VIT_CONV_MAX_KERNEL 16   /* Conv2d kernel size k */
#define B200VIT_POOL_MAX_KERNEL 16   /* MaxPool2d kernel size */
#define B200VIT_SEQ_POOL_MAX_DIM 1024  /* embedding width D of b200vit_seq_pool */
#define B200VIT_ATTN_KV_MAX_KEYS 16384  /* keys per image of b200vit_attention_kv */

/* what b200vit_cross_embed_nchw (CrossFormer's stage-1 cross-scale embedding) is built for */
#define B200VIT_CROSS_EMBED_MAX_SCALES 4     /* convolutions (scales) per call */
#define B200VIT_CROSS_EMBED_MAX_KERNEL 32    /* kernel size k of a scale */
#define B200VIT_CROSS_EMBED_MAX_CHANNELS 4   /* image channels C */
#define B200VIT_CROSS_EMBED_MAX_STRIDE 8     /* the shared stride s */
#define B200VIT_CROSS_EMBED_MAX_WIDTH 64     /* output channels n of a scale (a multiple of 8) */

/* what b200vit_attention_wide (the soft-split attention of T2T-ViT, one head as wide as the token) is built for */
#define B200VIT_ATTN_WIDE_MAX_TOKENS 1024  /* tokens n per image */
#define B200VIT_ATTN_WIDE_MAX_WIDTH 4096   /* padded head width dp */

/* what b200vit_ats_select (Adaptive Token Sampling's token selection) is built for */
#define B200VIT_ATS_MAX_TOKENS 4096         /* row slot S_in per image */
#define B200VIT_ATS_MAX_HEAD_TOKENS 16384   /* H * S_in: the per-head scores and value norms held in shared memory */

const char* b200vit_last_error(void);
int b200vit_version(void);
/* number of kernels this library has launched in the calling process (all threads) since load / last reset */
int64_t b200vit_launch_count(void);
void b200vit_reset_launch_count(void);
/* 0 when device `dev` is sm_90 and the driver entry points the library needs resolve; negative otherwise */
int b200vit_device_ok(int dev);

/*
 * out[M, N] = epilogue( A[M, K] (bf16, row stride lda) x W[N, K]^T (bf16, row stride ldw) ), fp32 accumulate.
 * TMA-fed wgmma GEMM, persistent, warp specialised (one loader and two consumer warpgroups; the loaders also stage the
 * residual tile, bias, col_s and LN-fold row sums in shared memory ahead of the epilogue).  Replaces every nn.Linear on the path:
 *   vit.py:20,23 (FeedForward), vit.py:44,47 (to_qkv / to_out), vit.py:102 (patch projection), vit.py:116 (mlp_head);
 *   simple_vit.py:30,32,47,48,93,108.
 * out_bf16 and/or out_f32 (either may be NULL, not both), row stride ldo (elements).
 * EPI_LNFOLD: ln_sums[M][ln_parts][2] = per-row PARTIAL (sum, sum of squares) of A (added up in index order, so the
 *             result is deterministic), ln_dim = K, col_s[N] = sum_k W[n,k] (fp32).
 * EPI_STATS:  stats_out[M][P][2], P = b200vit_stats_parts(N): every slot is written exactly once (no atomics).
 * Requirements: A, W 16-byte aligned, lda, ldw multiples of 8 and >= K.  Any K >= 1: the operands are read through
 * TMA, which zero-fills columns K .. of a k block, so columns past K of A and W are never read (T2T-ViT's soft splits
 * run at K = the true width w, e.g. 147 or 1323).
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
 * Shifted patch tokenization + LayerNorm(5*C*p*p) (SPT, vit_for_small_dataset.py:81-96): img[B, C, H, W] (bf16, NCHW
 * contiguous) -> A[B*gh*gw, ldo] bf16 with, for k = 0..4,
 *   A[b*(gh*gw) + h*gw + w, (p1*p + p2)*5C + k*C + c] = LN_over_patch(src_k[b, c, h*p + p1, w*p + p2]) * gamma + beta
 *   src_0(y, x) = img(y, x), src_1 = img(y, x-1), src_2 = img(y, x+1), src_3 = img(y-1, x), src_4 = img(y+1, x),
 * zero outside the image: the concat of the image and its four one-pixel shifts (F.pad by (1,-1,0,0), (-1,1,0,0),
 * (0,0,1,-1), (0,0,-1,1)), cut into '(p1 p2 c)' patches over 5C channels, without materialising either.  Columns
 * [5*C*p*p, ldo) are zero filled (K padding for the GEMM).  ldo multiple of 8, out_bf16 16-byte aligned.
 */
int b200vit_patchify_spt_ln(const void* img, const float* gamma, const float* beta, void* out_bf16, int64_t ldo, int B,
                            int C, int H, int W, int p, float eps, void* stream);

/*
 * Token assembly after the patch projection: y[B*n, D] (fp32, patch GEMM output incl. bias) ->
 *   x[b, t, :] = LN_D(y[b, t - ncls, :]) * gamma + beta + pos[t, :]   for t >= ncls
 *   x[b, 0, :] = cls[:] + pos[0, :]                                    if ncls == 1
 *   x[b, ncls + n + r, :] = tail[r, :]                                 for r < ntail (register tokens, no pos;
 *                                                                       simple_vit_with_register_tokens.py:124-126)
 * written as the fp32 residual stream x[B*(ncls+n+ntail), D].  Optional (may be NULL): xb_bf16 = bf16 copy of x and
 * stats[M][2] = per-row (sum, sum of squares) of that copy -- the inputs of the first LN-folded GEMM.
 * Replaces nn.LayerNorm(dim) vit.py:103, cls concat vit.py:122-123, pos add vit.py:125-127 (simple_vit.py:94,114).
 * pos == NULL: no positional term at all (the rotary ViTND, vit_nd_rotary.py:272-287, positions act on q / k instead).
 * gamma == NULL: no LayerNorm, the patch rows are y itself (beta is ignored; SPT has no LayerNorm(dim),
 * vit_for_small_dataset.py:127-132).  Applies to b200vit_embed_tokens_grouped as well.
 */
int b200vit_embed_tokens(const float* y, const float* gamma, const float* beta, const float* cls, const float* pos,
                         const float* tail, float* x, void* xb_bf16, float* stats, int B, int n, int ncls, int ntail,
                         int D, float eps, void* stream);
/*
 * The same assembly over `groups` token groups (y holds groups*n patch rows) whose positional rows come from a block of
 * a larger table: group g reads the block starting at row (g % pos_period) * pos_stride.  Within the block, patch t
 * reads row ncls + t and cls row c row c when cls_pos != 0; with cls_pos == 0 patch t reads row t and the cls rows
 * get no position.  ViViT's [F'max, n_max] table sliced to [:frames, :n] (vivit.py:227-231): groups = B*F',
 * pos_period = F', pos_stride = n_max, cls_pos = 0.  b200vit_embed_tokens is this call with (1, 0, 1).
 */
int b200vit_embed_tokens_grouped(const float* y, const float* gamma, const float* beta, const float* cls,
                                 const float* pos, const float* tail, float* x, void* xb_bf16, float* stats, int groups,
                                 int n, int ncls, int ntail, int D, float eps, int pos_period, int pos_stride,
                                 int cls_pos, void* stream);

/*
 * N-d patchify without a LayerNorm (vit_nd.py:130-145 / vit_nd_rotary.py:216-231, 'b c (f p0) (g p1) ... ->
 * b (f g ...) (p0 p1 ... c)'): img[B, C, S_0 .. S_{r-1}] (bf16, contiguous), rank r = 1..7, patch[i] dividing shape[i]
 * (shape / patch: HOST int arrays of r entries) -> A[B*n, ldo] bf16, n = prod(S_i / p_i), with
 *   A[b*n + rowmajor(g_0 .. g_{r-1}), rowmajor(q_0 .. q_{r-1})*C + c] = img[b, c, g_0*p_0 + q_0, ..., g_{r-1}*p_{r-1} + q_{r-1}]
 * as bit copies.  Columns [C * prod(p_i), ldo) are zero filled (K padding for the GEMM).  ldo multiple of 8, out_bf16
 * 16-byte aligned.
 */
int b200vit_patchify_nd(const void* img, void* out_bf16, int64_t ldo, int B, int C, int rank, const int* shape,
                        const int* patch, void* stream);

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
 * dh = 32, 64, 80 (canonical ViT-H/14) or 128; a head is split into 64- and 16-column slabs (a 96-wide head would
 * fall out of the same scheme as 64 + 2 x 16, but is not built).
 * 128 < N <= 256 with dh = 32 or 64 (ViT-B/16 and ViT-L/16 at 224^2: 197 tokens) runs a persistent kernel instead: one
 * CTA per SM loops over (sequence, head) items, each head's Q, K and V are staged in shared memory once while the
 * next head loads underneath, four warpgroups take 64 query rows each, the last key block runs at its real width
 * rounded up to 16 keys, and the output leaves through TMA stores.  It keeps the per-block arithmetic and its order,
 * so both kernels give the same bits.  dh = 80 and 128 do not fit two heads in shared memory and, like calls with
 * B200VIT_ATTN_MASK_SELF, keep the tiled kernel at every N.
 * Isolation (this and every attention entry point below): each sequence's output is computed from its own rows only,
 * so a NaN or Inf in one sequence (image, packed sequence, batch element of b200vit_attention_axial) leaves every other
 * sequence's output bit-identical, and no row past the buffer's addressed rows is read.
 */
int b200vit_attention(const void* qkv, void* out, int B, int N, int H, int dh, float scale, void* stream);
/* ... with flags: B200VIT_ATTN_MASK_SELF excludes each query's own key (masked_fill(eye, -finfo.max),
 * vit_for_small_dataset.py:53-57; a sequence of one token keeps it, as that fill does).  b200vit_attention is this call
 * with flags = 0. */
int b200vit_attention_ex(const void* qkv, void* out, int B, int N, int H, int dh, float scale, int flags, void* stream);

/*
 * Variable-length attention over PACKED sequences (any length): tokens [cu_seqlens[s], cu_seqlens[s+1]) of
 * qkv[total_tokens, 3*H*dh] attend only among themselves; out[total_tokens, H*dh].  This is the block-diagonal
 * "same image" attention of NaViT (na_vit.py:335-337 mask + 161-166 SDPA) without padding or an O(L^2) mask, and the
 * long-sequence (N > 512) path of ViT.  dh = 32, 64, 80 or 128, and 160 without B200VIT_ATTN_MASK_SELF (the one head of a
 * T2T-ViT soft-split layer up to 160 wide, t2t.py:40 / vit.py Attention, 2 x 64 + 2 x 16 column slabs).  cu_seqlens_dev[num_seqs+1] and tile_prefix_dev[num_seqs+1] (number of 128-row
 * query tiles before sequence s; tile_prefix[num_seqs] == total_tiles) are DEVICE int32 arrays built by the caller.
 */
int b200vit_attention_varlen(const void* qkv, void* out, const int32_t* cu_seqlens_dev, const int32_t* tile_prefix_dev,
                             int num_seqs, int total_tokens, int total_tiles, int H, int dh, float scale,
                             void* stream);
/* ... with flags as b200vit_attention_ex (indices within each sequence); b200vit_attention_varlen is flags = 0. */
int b200vit_attention_varlen_ex(const void* qkv, void* out, const int32_t* cu_seqlens_dev,
                                const int32_t* tile_prefix_dev, int num_seqs, int total_tokens, int total_tiles, int H,
                                int dh, float scale, int flags, void* stream);

/*
 * Softmax attention over short strided sequences with an optional key mask (ViViT's temporal attention,
 * vivit.py:144-150, and its masked temporal transformer, vivit.py:75-100,268):
 *   qkv[B*L*G, 3*H*dh] bf16 packed as for b200vit_attention; out[B*L*G, H*dh] bf16.
 *   Token j of sequence s = b*G + p is row b*L*G + j*G + p of both (G = 1: B contiguous sequences of L tokens).
 *   key_mask: NULL, or a DEVICE uint8 [B][L] array (1 = keep) shared by the G sequences of batch element b.
 * A query row whose keys are all masked gets 0 when zero_masked_rows != 0 (scaled_dot_product_attention with a boolean
 * mask) and the mean of the L values of its sequence otherwise (masked_fill(-finfo.max) before the softmax).
 * L <= 64, dh = 32, 64, 80 or 128; qkv and out 16-byte aligned.  Rows of out outside the addressed set are untouched.
 */
int b200vit_attention_axial(const void* qkv, void* out, const uint8_t* key_mask, int B, int L, int G, int H, int dh,
                            float scale, int zero_masked_rows, void* stream);

/*
 * Softmax attention inside non-overlapping p x p windows of a token map (Twins-SVT's locally-grouped attention,
 * twins_svt.py:85-120): B maps of gh x gw tokens, token (b, y, x) at row (b*gh + y)*gw + x of
 *   qkv[B*gh*gw, 3*H*dh] bf16 packed as for b200vit_attention; out[B*gh*gw, H*dh] bf16.
 * Window (b, wy, wx) is the p*p rows (b*gh + wy*p + i)*gw + wx*p + j, i, j < p; each head attends among them and the
 * result goes back to the same rows.  One 64-row tile holds as many whole windows of one image as fit (1 for p >= 6,
 * 64 for p = 1).  p*p <= 64, gh and gw multiples of p, dh = 32, 64, 80 or 128; qkv and out 16-byte aligned.
 * Isolation: a window's output is computed from its own rows only and nothing outside the B*gh*gw rows is read or
 * written.  A NaN or Inf stays within its image, and within its window when the window has a tile of its own
 * (p*p > 32); windows that share a tile give each other's values the probability 0, so any finite change in one
 * leaves the others bit-identical.
 */
int b200vit_attention_window(const void* qkv, void* out, int B, int gh, int gw, int p, int H, int dh, float scale,
                             void* stream);

/*
 * Attention of every query of an image over keys and values that live in another buffer and have another length
 * (Twins-SVT's global sub-sampled attention, twins_svt.py:122-157, where they come from a strided convolution):
 *   q[B*Nq, H*dh] bf16 (row stride ldq), kv[B*Nk, 2*H*dh] bf16 packed k | v (row stride ldkv), both head-major;
 *   out[B*Nq, H*dh] bf16 (contiguous) = softmax(scale * q k^T) v per image and head.
 * 128-row query tiles, keys in blocks of 64 with an fp32 online softmax, both products on wgmma, keys past Nk masked.
 * When the key blocks of an (image, head) fit in shared memory they are loaded once per CTA and the CTA's query tiles
 * loop over them (up to 1024 / 704 / 576 / 320 keys for dh = 32 / 64 / 80 / 128); longer key sets stream through a
 * ring of block slots once per query tile.  Nq >= 1, 1 <= Nk <= B200VIT_ATTN_KV_MAX_KEYS (Nk = 1: out is that value
 * row), dh = 32, 64, 80 or 128, B and H <= 65535; ldq and ldkv multiples of 8; q, kv and out 16-byte aligned.  Each
 * image's output is computed from its own rows only, and no row past B*Nq or B*Nk is read.
 */
int b200vit_attention_kv(const void* q, int64_t ldq, const void* kv, int64_t ldkv, void* out, int B, int Nq, int Nk,
                         int H, int dh, float scale, void* stream);

/*
 * b200vit_attention_kv with a key count per image: image b attends over its first nk[b] keys (clamped to [1, Nk]) of
 * its Nk-row slot, nk_dev a DEVICE int32 [B] array (Adaptive Token Sampling: the kept queries over the image's valid
 * keys, ats_vit.py:142-150 and 160, whose padded keys get probability 0).  Rows of the slot past nk[b] inside its last
 * 64-key block are loaded with probability exactly 0, so only a NaN or Inf there (which can come only from the same
 * image) reaches the image's output; no row outside the image's slot is read.  out must overlap neither q nor kv.  Everything else (layout, limits,
 * isolation, dh = 32, 64, 80 or 128) as b200vit_attention_kv, which stays a separate instance and gives the same bits
 * as before.
 */
int b200vit_attention_kv_lens(const void* q, int64_t ldq, const void* kv, int64_t ldkv, void* out, int B, int Nq,
                              int Nk, const int32_t* nk_dev, int H, int dh, float scale, void* stream);

/*
 * b200vit_attention_kv with key heads of another width than the value heads (ScalableViT's SSA,
 * scalable_vit.py:71-124, where dim_key and dim_value are separate hyperparameters):
 *   q[B*Nq, H*dk] bf16 (row stride ldq), kv[B*Nk, H*dk + H*dv] bf16 packed k | v (row stride ldkv), head-major;
 *   out[B*Nq, H*dv] bf16 (contiguous) = softmax(scale * q k^T) v per image and head.
 * dk = 16, 32, 48 or 64; dv = 32 or 64.  A dim_key that is a multiple of 8 runs at the next multiple of 16: the caller
 * inserts zero columns per head in q and k (zero rows of their projection weights), which add exactly 0 to every score,
 * and passes the scale of the unpadded width.  out must overlap neither q nor kv.  Everything else (tiling, limits,
 * checks, isolation) as b200vit_attention_kv, which is this call with dk = dv = dh (dh = 32, 64, 80 or 128).
 */
int b200vit_attention_kv_ex(const void* q, int64_t ldq, const void* kv, int64_t ldkv, void* out, int B, int Nq, int Nk,
                            int H, int dk, int dv, float scale, void* stream);

/*
 * Attention with a learned relative-position bias over an F x F token map (LeViT, levit.py:40-108):
 *   qkv[B*F*F, ld] bf16, token (b, y, x) at row (b*F + y)*F + x; columns q (H*dk) | k (H*dk) | v (H*dv), head-major.
 *   Queries are the tokens (s*i, s*j), i, j < Fq = ceil(F / s), s = 1 or 2 (the downsampling attention's stride-2
 *   to_q, gathered from the same full-grid qkv).
 *   out[B*Fq*Fq, H*dv] bf16 (contiguous), row (b*Fq + i)*Fq + j:
 *     softmax_j(scale * q.k_j + table[h][|dy|*F + |dx|]) v,  (dy, dx) the offset between the query's and key j's
 *     positions on the F x F grid.  table fp32 [H][F*F] (the caller passes pos_bias.weight^T / scale).
 *   flags: B200VIT_ATTN_GELU_OUT applies exact-erf GELU to each output before rounding.
 * One CTA per 64 queries of an (image, head); keys and values stream through two shared-memory slots in blocks of 64,
 * fp32 online softmax, both products on wgmma.  dk = 16, 32 or 64; dv = 32, 64 or 128; F*F <=
 * B200VIT_ATTN_POSBIAS_MAX_KEYS; ld a multiple of 8; qkv, out and table 16-byte aligned; B and H <= 65535.
 * Isolation as b200vit_attention: each image's output is computed from its own rows only, no row past B*F*F is read,
 * and no output row outside the B*Fq*Fq addressed is written.
 */
int b200vit_attention_posbias(const void* qkv, int64_t ld, void* out, const float* table, int B, int F, int s, int H,
                              int dk, int dv, float scale, int flags, void* stream);

/*
 * MaxViT's window attention with a relative-position bias (max_vit.py:121-206) over B maps of gh x gw tokens, token
 * (b, y, x) at row (b*gh + y)*gw + x of qkv[B*gh*gw, 3*H*dh] bf16 (packed as for b200vit_attention) and of
 * out[B*gh*gw, H*dh] bf16.  With X = gh / w and Y = gw / w windows along each axis, window (b, i, j) holds the w*w
 * tokens of local coordinates (u, v), u, v < w, at map position
 *   grid = 0 (block, 'b d (x w1) (y w2)'):  (i*w + u, j*w + v)
 *   grid = 1 (grid,  'b d (w1 x) (w2 y)'):  (u*X + i, v*Y + j)
 * and each head attends among them:  softmax_k(scale * q.k + table[h][(du + w-1)*(2w-1) + (dv + w-1)]) v,  (du, dv)
 * the query's local coordinates minus the key's.  table fp32 [H][(2w-1)^2] = rel_pos_bias.weight^T.
 * One CTA per (window, head): the window's rows are gathered with cp.async into one 64-row tile, the head's bias
 * table is staged in shared memory, both products on wgmma, an fp32 softmax over the w*w keys.
 * 1 <= w <= 8, gh and gw multiples of w, dh = 32, 64, 80 or 128, H <= 65535; qkv, out and table 16-byte aligned.
 * Isolation: a window's output is computed from its own rows only and nothing outside the B*gh*gw rows is read or
 * written; a NaN or Inf stays within its window.
 */
int b200vit_attention_window_relpos(const void* qkv, void* out, const float* table, int B, int gh, int gw, int w,
                                    int grid, int H, int dh, float scale, void* stream);

/* rows of the token map one CTA of b200vit_mbconv_dwconv sums per (image, channel): the partial sums have
 * ceil(oh*ow / B200VIT_MBCONV_PART_ROWS) parts per image */
#define B200VIT_MBCONV_PART_ROWS 64

/*
 * MBConv's depthwise 3 x 3 convolution + BatchNorm + GELU (max_vit.py:106-108) on B channels-last maps:
 *   x[B*h*w, C] bf16 -> y[B*oh*ow, C] bf16, oh = ceil(h / stride), ow = ceil(w / stride), zero padding 1,
 *   y = GELU_erf(bias[c] + sum_taps w9[tap][c] * x),  w9 fp32 [9][C] tap-major and bias fp32 [C] with the BatchNorm
 *   folded in by the caller.
 * part[B][P][C] fp32, P = ceil(oh*ow / B200VIT_MBCONV_PART_ROWS): part[b][p][c] = the sum of the bf16-rounded y of
 * rows p*PART_ROWS .. of image b in channel c, each slot written once in a fixed order (no atomics), so repeated calls
 * give the same bits.  stride 1 or 2; C a multiple of 8; all pointers 16-byte aligned; x and y do not overlap.
 */
int b200vit_mbconv_dwconv(const void* x, int64_t M, const float* w9, const float* bias, void* y, float* part, int B,
                          int h, int w, int C, int stride, void* stream);
/* ... with the activation `act` = B200VIT_EPI_GELU or B200VIT_EPI_SILU (y / (1 + exp(-y)), MobileViT's MV2Block,
 * mobile_vit.py:108-127, as the GEMM's EPI_SILU computes it), and `part` optional: NULL skips the channel sums
 * (MobileViT has no squeeze-excitation).  b200vit_mbconv_dwconv is this call with B200VIT_EPI_GELU and `part`
 * required; both give the same bits. */
int b200vit_mbconv_dwconv_ex(const void* x, int64_t M, const float* w9, const float* bias, void* y, float* part, int B,
                             int h, int w, int C, int stride, int act, void* stream);

/* tokens per group b200vit_attention_groups takes, (gh/ph)*(gw/pw) */
#define B200VIT_ATTN_GROUPS_MAX_TOKENS 4096

/*
 * MobileViT attention over strided patch groups (mobile_vit.py:64-72, 150-152):  B channels-last token maps of
 * gh x gw tokens, token (b, y, x) at row (b*gh + y)*gw + x of qkv[B*gh*gw, 3*H*dh] (packed q | k | v, head-major, as
 * for b200vit_attention) and of out[B*gh*gw, H*dh].  Group (b, i, j), i < ph, j < pw, is the set of tokens
 * (y'*ph + i, x'*pw + j); each head attends only within its group and each result goes back to the token's own row:
 *   out = softmax(scale * q k^T) v  over the group's (gh/ph)*(gw/pw) tokens.
 * Rows are gathered by this address map; no token is copied into group order.  ph = pw = 1 with gw = 1 gives B
 * contiguous sequences of gh tokens.
 * Numerics as b200vit_attention: scores q.k * scale in fp32, an fp32 online softmax over 64-key blocks with exp2 and
 * scale*log2(e) folded in, probabilities rounded to bf16 before P V, fp32 accumulation, one bf16 rounding of the
 * output.  mma.sync m16n8k8 for Q K^T and for P V (8 keys per MMA); one CTA stages one head's K and V of one or more groups in
 * shared memory once.
 * dh = 8 only; any H >= 1 (<= 65535); gh % ph == gw % pw == 0; 1 <= group length <= B200VIT_ATTN_GROUPS_MAX_TOKENS;
 * qkv and out 16-byte aligned.
 * Isolation: a group's output is computed from its own rows only; a NaN or Inf stays within its group; nothing outside
 * the B*gh*gw rows is read or written; repeated calls give the same bits.
 */
int b200vit_attention_groups(const void* qkv, void* out, int B, int gh, int gw, int ph, int pw, int H, int dh,
                             float scale, void* stream);

/*
 * SepViT's window attention with a window token (sep_vit.py:139-168) over B maps of gh x gw tokens, token (b, y, x) at
 * row (b*gh + y)*gw + x of qkv[B*gh*gw, 3*H*dh] bf16 (packed as for b200vit_attention) and of out[B*gh*gw, H*dh] bf16.
 * Window (b, wy, wx) of the (gh/p) x (gw/p) grid holds the p*p tokens (wy*p + u, wx*p + v) and one more token whose
 * q | k | v is tok_qkv[3*H*dh] bf16 (the layer's to_qkv applied to its window_tokens parameter, the same for every
 * window); each head attends among these p*p + 1 tokens:  softmax(scale * q k^T) v.  The window's own tokens' results
 * go to their rows of out; if tok_out is not NULL, the window token's result goes to row (b*(gh/p) + wy)*(gw/p) + wx
 * of tok_out[B*(gh/p)*(gw/p), H*dh] bf16, the reference's '(b x y)' window order.
 * One CTA per (window, head): row 0 of the 64-row tile is the window token, rows 1 .. p*p the window's tokens gathered
 * with cp.async; both products on wgmma.  Numerics as b200vit_attention_window: fp32 scores, exp2 with scale*log2(e)
 * folded in, probabilities rounded to bf16, fp32 accumulation, one bf16 rounding of the output.
 * p*p + 1 <= 64 (p <= 7), gh and gw multiples of p, dh = 32, 64, 80 or 128, H <= 65535; every pointer 16-byte aligned.
 * Isolation: a window's outputs are computed from its own rows and tok_qkv only and nothing outside the B*gh*gw rows
 * of qkv / out and the addressed rows of tok_out is read or written; a NaN or Inf stays within its window.
 */
int b200vit_attention_window_token(const void* qkv, const void* tok_qkv, void* out, void* tok_out, int B, int gh,
                                   int gw, int p, int H, int dh, float scale, void* stream);

/*
 * SepViT's attention across windows (sep_vit.py:182-205), out of place on B maps laid out as for
 * b200vit_attention_window_token, with nw = (gh/p)*(gw/p) windows per map:
 *   wqk[B*nw, 2*H*dh] bf16, row b*nw + j the window-token projection of window j of image b; head h's query is columns
 *   [2h*dh, 2h*dh + dh) and its key [2h*dh + dh, 2(h+1)*dh) (the per-head interleave of 'b (h c) n -> b h n c' then
 *   .chunk(2, -1));
 *   P = softmax_j(scale * wq_i . wk_j) per (image, head), over the nw windows;
 *   out[(window i, position w)] = sum_j P_ij o[(window j, position w)]  for every window position w < p*p, o and out
 *   [B*gh*gw, H*dh] bf16, head h's columns [h*dh, (h+1)*dh).
 * One CTA per (image, head, slice of up to 8 window positions): S = wq wk^T on one 64 x 64 wgmma and the softmax once,
 * then per position the nw rows of o through a two-buffer cp.async ring and O_w = P V_w on wgmma.  Numerics as
 * b200vit_attention_window_token.
 * 2 <= nw <= 64, gh and gw multiples of p, dh = 32, 64, 80 or 128; out != o; every pointer 16-byte aligned.
 * Isolation: an (image, head)'s output is computed from its own rows of wqk and o only, and nothing outside the
 * B*nw rows of wqk and the B*gh*gw rows of o / out is read or written; a NaN or Inf stays within its image and head.
 */
int b200vit_window_mix(const void* wqk, const void* o, void* out, int B, int gh, int gw, int p, int H, int dh,
                       float scale, void* stream);

/*
 * RegionViT's region-to-local attention (regionvit.py:167-176) over one buffer of both token maps of B images:
 * qkv[B*lh*lw + B*rh*rw, 3*H*dh] bf16 (packed as for b200vit_attention) holds the local tokens first, token (b, y, x)
 * at row (b*lh + y)*lw + x, then the region tokens, token (b, i, j) at row B*lh*lw + (b*rh + i)*rw + j; out
 * [same rows, H*dh] bf16 has the same layout.  Window (b, i, j) is the region token (b, i, j) and the wh x ww local
 * tokens (i*wh + u, j*ww + v), wh = lh/rh, ww = lw/rw; per head its n = 1 + wh*ww tokens attend together,
 *   softmax(scale * q k^T + bias) v,
 * bias = table[h*(2W-1)^2 + (u1-u2 + W-1) + (v1-v2 + W-1)*(2W-1)] between local tokens (u1, v1) (query) and (u2, v2)
 * (key), 0 for every pair that involves the region token.  table fp32 [H][(2W-1)^2] is the transposed
 * local_rel_pos_bias.weight of an R2LTransformer built with window_size W.  Each result goes to its own row of out.
 * One CTA per (window, head, 64-row query tile): the window's <= 4 key / value blocks gathered with cp.async, both
 * products on wgmma.  Numerics as b200vit_attention_window_relpos: fp32 scores, exp2 with scale*log2(e) folded in,
 * probabilities rounded to bf16, fp32 accumulation, one bf16 rounding of the output.
 * dh = 32, lh % rh == 0, lw % rw == 0, wh <= W, ww <= W, wh*ww + 1 <= 256, H <= 65535; every pointer 16-byte aligned.
 * Isolation: a window's outputs are computed from its own rows only and nothing outside the B*(lh*lw + rh*rw) rows
 * of qkv / out is read or written; a NaN or Inf stays within its window.
 */
int b200vit_attention_region_local(const void* qkv, void* out, const float* table, int B, int lh, int lw, int rh,
                                   int rw, int W, int H, int dh, float scale, void* stream);

/*
 * Squeeze-excitation around two bias-free GEMMs (max_vit.py:47-62):
 *   b200vit_se_pool:   pooled[b][c] bf16 = (sum_p part[b][p][c]) * inv_n, the parts added in index order (the mean of
 *                      b200vit_mbconv_dwconv's output); the gate then runs as GEMM(EPI_SILU), GEMM(EPI_SIGMOID) over
 *                      the B pooled rows, so each SE weight matrix is read once per batch
 *   b200vit_se_scale:  h[b*n + t][c] = bf16(h[b*n + t][c] * gate[b][c]), in place, gate bf16 [B][C]
 * C a multiple of 8; all pointers 16-byte aligned.
 */
int b200vit_se_pool(const float* part, void* pooled, int B, int P, int C, float inv_n, void* stream);
int b200vit_se_scale(void* h, const void* gate, int B, int n, int C, void* stream);

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
 * dh = 32, 64, 80 or 128 (this and every head-norm / pooling entry point below).
 */
int b200vit_qk_rmsnorm(void* qkv, const float* gamma_qk, int T, int H, int dh, void* stream);

/*
 * Linear + per-head RMSNorm in one pass (NaViT to_q / to_kv followed by q_norm / k_norm, na_vit.py:145-150):
 *   out[M, N] bf16 = epilogue(A W^T)   with flags in {EPI_BIAS, EPI_LNFOLD} exactly as b200vit_gemm_bf16, then the first
 *   norm_heads heads (dh columns each, from column 0; norm_heads * dh <= N) of every row are replaced by
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
 * Golden-gate N-d rotary embedding of q and k, in place on the packed qkv[T, 3*H*dh] buffer (v untouched;
 * GoldenGateRoPENd.forward, vit_nd_rotary.py:74-96, applied at :143-147).  cs fp32 [R][H][dh/2][2] = (cos, sin) of
 * theta; token t uses table row t % R (R = N: every image shares one patch grid; R = T: positions given per token).
 * For every head and f < dh/2, with x = head[f], y = head[f + dh/2]:
 *   x' = x cos - y sin,   y' = x sin + y cos
 * in fp32 with every product and sum rounded on its own (no FMA), then rounded to bf16: bit-identical to the
 * reference's expression for the same bf16 q / k and the same table.  qkv and cs 16-byte aligned.
 */
int b200vit_rope_qk(void* qkv, const float* cs, int R, int T, int H, int dh, void* stream);

/*
 * The same normalisation on any row-major bf16 buffer: the `nheads` consecutive dh-wide heads that start at column 0
 * of every row buf[t*ld ...] (the k half of a [k | v] buffer for the attention pooling, na_vit.py:143-150);
 * gamma fp32 [nheads][dh].  ld in elements, multiple of 8; buf 16-byte aligned.
 */
int b200vit_rmsnorm_heads(void* buf, int64_t ld, const float* gamma, int T, int nheads, int dh, void* stream);
/* ... and its LayerNorm (no bias) flavour: (v - mean) * rsqrt(var + eps) * gamma[h, d] over each dh-wide head. */
int b200vit_layernorm_heads(void* buf, int64_t ld, const float* gamma, int T, int nheads, int dh, float eps,
                            void* stream);
/* ... and with a shift and exact-erf GELU after it, SepViT's window-token pre-norm (sep_vit.py:96-98):
 *   v <- GELU_erf((v - mean) * rsqrt(var + eps) * gamma[d] + beta[d]),  gamma, beta fp32 [dh] shared by the heads,
 * statistics in fp32 with the two-pass variance.  In place on the nheads heads from column 0 of every row buf[t*ld
 * ...]; ld a multiple of 8, buf, gamma and beta 16-byte aligned.  Each row is read and written only by its own warp. */
int b200vit_head_layernorm_gelu(void* buf, int64_t ld, const float* gamma, const float* beta, int T, int nheads, int dh,
                                float eps, void* stream);

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

/*
 * Class-token cross attention (CrossViT, cross_vit.py:53-71 with kv_include_self = True): one query per image attends
 * over its own key / value and n context rows of the same image.  For image b < B and head h < H:
 *   out[b, h*dh:(h+1)*dh] = softmax_j(scale * q_bh . k_jh) v_jh,   j over {self} u {the n context rows of image b}
 *   qkv_self[B, 3*H*dh] bf16, packed q | k | v as for b200vit_attention: q, the self key and the self value of image b.
 *   ctx_kv: [k | v] rows 2*H*dh wide (row stride ctx_ld); image b's rows start at row b*ctx_rows_per_image + ctx_first
 *   (a kv GEMM over every row of the other stream, its cls rows skipped with ctx_first = 1).
 *   out: bf16 [B, H*dh], row stride ldo.
 * n = 0..16384 (n = 0: out = v_self), dh = 32, 48, 64, 80 or 128; softmax in fp32.  One CTA of 8 warps per (image, head):
 * the NaViT pooling kernel above with a per-image bf16 query and a strided context.  ctx_ld and ldo multiples of 8,
 * pointers 16-byte aligned; ctx_kv may be NULL when n = 0.
 */
int b200vit_attention_cls(const void* qkv_self, const void* ctx_kv, int64_t ctx_ld, int64_t ctx_rows_per_image,
                          int ctx_first, int n, void* out, int64_t ldo, int B, int H, int dh, float scale,
                          void* stream);

/*
 * Attention with the softmax probabilities mixed across heads: DeepViT's re-attention (deepvit.py:56-67).  B sequences
 * of N tokens, qkv[B*N, 3*H*dh] bf16 packed as for b200vit_attention, out[B*N, H*dh] bf16.  Per sequence, for query i,
 * key j and heads g, f < H:
 *   s_g[i,j] = scale * q_g[i] . k_g[j]
 *   p_g      = softmax_j(s_g)
 *   p'_f     = sum_g post[g][f] p_g
 *   p''_f    = gamma_f (p'_f - mean) / sqrt(var + eps) + beta_f, mean / var over the H values p'_. of (i, j)
 *                                                      (head_ln_gamma NULL: p'' = p')
 *   out_f[i] = sum_j p''_f[i,j] v_f[j]
 * post: device fp32 [H][H], indexed [input head][output head] (the einsum 'b h i j, h g -> b g i j');
 * head_ln_gamma / head_ln_beta: device fp32 [H], both or neither, eps > 0.  Mixing, softmax and the LayerNorm run in
 * fp32; QK^T and PV on wgmma.  No score or probability tile goes to global memory: each CTA holds the score tiles of
 * every head for 64 query rows and recomputes them per group of output heads (QK^T costs 3 ceil(H / 2G) times that of
 * plain attention, G = 1..4 output heads per warpgroup, see csrc/headmix.cu).  N = 1..16384, dh = 32, 48, 64,
 * 80 or 128, H <= 16, H*dh <= 1024, qkv and out 16-byte aligned.
 */
int b200vit_attention_headmix(const void* qkv, void* out, int B, int N, int H, int dh, float scale,
                              const float* post, const float* head_ln_gamma, const float* head_ln_beta,
                              float head_ln_eps, void* stream);

/*
 * b200vit_attention_headmix with talking heads before the softmax as well (CaiT, cait.py:92-101): the scores are mixed
 * across heads before the softmax,
 *   s'_g[i,j] = sum_h pre[h][g] s_h[i,j],   p_g = softmax_j(s'_g)
 * and the rest is as above.  pre: device fp32 [H][H], [input head][output head], or NULL (no pre-mix: exactly
 * b200vit_attention_headmix).  Keys beyond the sequence are masked after the mix.
 */
int b200vit_attention_headmix_ex(const void* qkv, void* out, int B, int N, int H, int dh, float scale,
                                 const float* pre, const float* post, const float* head_ln_gamma,
                                 const float* head_ln_beta, float head_ln_eps, void* stream);

/*
 * Class-token attention with talking heads (CaiT's class attention, cait.py:83-103 with a context): the addressing of
 * b200vit_attention_cls (qkv_self, strided ctx_kv rows, out row stride ldo), with the heads mixed before and after the
 * softmax.  For image b, key j over {self} u {the n context rows of image b}, heads g, f < H:
 *   s_h[j] = scale * q_h . k_h[j];   s'_g = sum_h pre[h][g] s_h;   p_g = softmax_j(s'_g);   p'_f = sum_g post[g][f] p_g
 *   out[b, f*dh:(f+1)*dh] = sum_j p'_f[j] v_f[j]
 * pre, post: device fp32 [H][H], [input head][output head], both required.  n = 0..16384, dh = 32, 48, 64, 80 or 128,
 * H <= 16, H*dh <= 1024; scores, softmax and both mixes in fp32.  One CTA of 8 warps per image.  ctx_ld and ldo
 * multiples of 8, qkv_self / ctx_kv / out 16-byte aligned; ctx_kv may be NULL when n = 0.
 */
int b200vit_attention_cls_headmix(const void* qkv_self, const void* ctx_kv, int64_t ctx_ld, int64_t ctx_rows_per_image,
                                  int ctx_first, int n, void* out, int64_t ldo, int B, int H, int dh, float scale,
                                  const float* pre, const float* post, void* stream);

/*
 * Cross-covariance attention (XCiT's XCA, xcit.py:109-148): attention over the dh channels of each head, not over its
 * tokens.  qkv[B*N, 3*H*dh] bf16 packed as for b200vit_attention; tau: device fp32 [H] (temperature.exp()).  For image
 * b and head h, with q, k, v its [N, dh] slices:
 *   G = q^T k,  A_ij = softmax_j(tau_h G_ij / (max(|q_:,i|, 1e-12) max(|k_:,j|, 1e-12))),  out_ni = sum_j A_ij v_nj
 * (F.normalize's eps rule: an all-zero q or k column gives zero scores, never NaN).  out[B*N, H*dh] bf16, (h d) column
 * order.  The cost is linear in N; accumulation, norms and softmax are fp32 with fixed summation orders and no atomics,
 * so repeated calls give the same bits.  One CTA per (image, head).  N = 1..16384, dh = 32, 48, 64, 80 or 128,
 * H*dh a multiple of 8, qkv and out 16-byte aligned.
 */
int b200vit_attention_xca(const void* qkv, const float* tau, void* out, int B, int N, int H, int dh, void* stream);

/*
 * Local patch interaction (XCiT's LPI, xcit.py:150-167) over B images of gh x gw tokens, out of place:
 *   y = x + conv2'(GELU(conv1'(LayerNorm(x))))
 * x, y: fp32 [B*gh*gw, D], token (b, r, c) at row b*gh*gw + r*gw + c; y must not overlap x (every token reads its
 * neighbours' rows of x).  LayerNorm: ln_gamma, ln_beta [D], ln_eps.  conv1', conv2': depthwise k x k, zero padding
 * k / 2, weights w1, w2 fp32 [k*k][D] (tap dy*k + dx major, channel minor) and biases b1, b2 [D]; the caller folds
 * BatchNorm (eval) into conv1' and LayerScale into conv2'.  Both paddings are zeros of the padded tensor: of the
 * LayerNorm output for conv1', of the GELU output for conv2'.  GELU is the erf form.
 * y_bf16 [M, D] bf16 and y_stats [M][2] fp32 (both, or both NULL): the bf16 copy of y and per row the (sum, sum of
 * squares) of that copy, exactly as b200vit_rowstats_cast writes them, for an LN-folded GEMM on y.
 * ln_scratch: fp32 [M][2] scratch (the LayerNorm statistics of x), overwritten.  k = 1, 3, 5 or 7; D a multiple of 4;
 * x, y 16-byte aligned, y_bf16 8-byte aligned.
 */
int b200vit_local_patch_interaction(const float* x, float* y, void* y_bf16, float* y_stats, float* ln_scratch,
                                    const float* ln_gamma, const float* ln_beta, float ln_eps, const float* w1,
                                    const float* b1, const float* w2, const float* b2, int B, int gh, int gw, int D,
                                    int k, void* stream);

/*
 * Overlapping patch extraction (PiT's nn.Unfold(kernel_size=p, stride=s) + Rearrange('b c n -> b n c'),
 * pit.py:140-147): img[B, C, H, W] bf16 (NCHW, contiguous) -> out[B*oh*ow, ldo] bf16, oh = (H - p) / s + 1,
 * ow = (W - p) / s + 1 (trailing pixels that do not fill a stride step are dropped), with
 *   out[b*oh*ow + r*ow + c, (ch*p + i)*p + j] = img[b, ch, r*s + i, c*s + j]
 * as bit copies (Unfold's column order: channel slowest).  Columns [C*p*p, ldo) are zero filled (K padding for the
 * GEMM).  p >= 2, s >= 1, H and W >= p; ldo a multiple of 8 and >= C*p*p; out_bf16 16-byte aligned.  Each CTA stages the
 * image rows of one patch row in shared memory, so a pixel covered by several patches of that row is read once.
 */
int b200vit_unfold_patches(const void* img, void* out_bf16, int64_t ldo, int B, int C, int H, int W, int p, int s,
                           void* stream);

/*
 * PiT's pooling layer up to its 1 x 1 convolution (Pool, pit.py:98-113): x[M, D] fp32 is the residual stream of B
 * images of 1 + h*w rows (row b*(1 + h*w) the cls row, then token r*w + c of the h x w grid; M = B*(1 + h*w)).
 *   a[b*(1 + oh*ow) + 1 + t, o] = bias[o] + sum_{dy, dx < 3} w9[dy*3 + dx][o] x_grid[b, 2*r - 1 + dy, 2*q - 1 + dx, o / 2]
 * for output token t = r*ow + q of the oh x ow = ceil(h / 2) x ceil(w / 2) grid and o < 2D: the depthwise 3 x 3,
 * stride 2, zero padding 1 convolution with channel multiplier 2 (Conv2d(D, 2D, 3, 2, 1, groups=D): output channel o
 * reads input channel o / 2), accumulated in fp32 and rounded to bf16 -- the A operand of the 1 x 1 convolution's GEMM.
 * Row b*(1 + oh*ow) of a (the cls slot) is zero filled, so one GEMM over all B*(1 + oh*ow) rows writes the next
 * stage's stream, whose cls rows cls_ff then overwrites.  cls[b, :D] = bf16 copy of x's cls row of image b: the A
 * operand of the cls_ff GEMM.  w9: fp32 [9][2D] (tap major, output channel minor), bias fp32 [2D].
 * D a multiple of 8; lda >= 2D and ldc >= D, multiples of 8; x, w9, bias, a_bf16, cls_bf16 16-byte aligned.  Each
 * image's outputs are computed from its own rows only, and repeated calls give the same bits.
 */
int b200vit_pit_pool(const float* x, int64_t M, int B, int h, int w, int D, const float* w9, const float* bias,
                     void* a_bf16, int64_t lda, void* cls_bf16, int64_t ldc, void* stream);

/*
 * The A operand of a zero-padded Conv2d(C, Cout, k, stride s, padding p) as a GEMM (CCT's tokenizer, cct.py:181-190),
 * oh = (H + 2p - k) / s + 1, ow = (W + 2p - k) / s + 1, one row per output pixel b*oh*ow + r*ow + q, written as bit
 * copies; a tap outside the image is zero and so are columns [K, ldo) (K padding for the GEMM).
 *   _nchw: img[B, C, H, W] bf16 (NCHW, contiguous), column (c*k + i)*k + j = img[b, c, r*s - p + i, q*s - p + j]
 *          (F.unfold's order: channel slowest, the layout of the Conv2d weight itself), K = C*k*k.  Each CTA stages the
 *          image rows one output row covers, zero halo included, in shared memory.
 *   _nhwc: x[M, C] bf16 channels-last (pixel (b, y, x) at row (b*H + y)*W + x, M = B*H*W), column (i*k + j)*C + c =
 *          x[(b, r*s - p + i, q*s - p + j), c] (channel fastest, 16-byte vectors: C a multiple of 8), K = k*k*C.  The
 *          caller permutes the weight to [Cout, k, k, C] to match.
 * 1 <= k <= B200VIT_CONV_MAX_KERNEL, s >= 1, 0 <= p < k, H + 2p and W + 2p >= k; ldo a multiple of 8 and >= K;
 * out_bf16 16-byte aligned (and x for _nhwc).
 */
int b200vit_conv_im2col_nchw(const void* img, void* out_bf16, int64_t ldo, int B, int C, int H, int W, int k, int s,
                             int p, void* stream);
int b200vit_conv_im2col_nhwc(const void* x, int64_t M, void* out_bf16, int64_t ldo, int B, int H, int W, int C, int k,
                             int s, int p, void* stream);
/* ... with x's rows ldx elements apart (ldx a multiple of 8, >= C): the channels-last map may be a column slice of a
 * wider buffer (MobileViT's concatenation, mobile_vit.py:155-157).  b200vit_conv_im2col_nhwc is this call with
 * ldx = C. */
int b200vit_conv_im2col_nhwc_ex(const void* x, int64_t ldx, int64_t M, void* out_bf16, int64_t ldo, int B, int H,
                                int W, int C, int k, int s, int p, void* stream);

/*
 * Patch merging + LayerNorm between the stages of a hierarchical model (Twins-SVT's PatchEmbedding up to its 1 x 1
 * convolution, twins_svt.py:59-75): x[M, C] fp32 is the token map of B images of gh x gw tokens (token (b, y, x) at
 * row (b*gh + y)*gw + x, M = B*gh*gw); output row b*(gh/p)*(gw/p) + oy*(gw/p) + ox holds the p x p block's tokens,
 *   out[row, (p1*p + p2)*C + c] = LN(x[(b, oy*p + p1, ox*p + p2), c]) * gamma[(p1*p + p2)*C + c] + beta[...],
 * the LayerNorm over all p*p*C values of the row (fp32, biased variance, eps inside the square root), rounded to bf16:
 * the A operand of the convolution's GEMM.  The reference orders the merged features (c p1 p2); the caller permutes
 * its gamma, beta and weight columns to (p1 p2 c), the order of contiguous reads.  Columns [p*p*C, ldo) are zero
 * filled (K padding).  gh and gw multiples of p, C a multiple of 4; ldo a multiple of 8 and >= p*p*C; x, gamma, beta
 * and out_bf16 16-byte aligned.
 */
int b200vit_merge_patches_ln(const float* x, int64_t M, const float* gamma, const float* beta, void* out_bf16,
                             int64_t ldo, int B, int gh, int gw, int C, int p, float eps, void* stream);

/*
 * Positional encoding generator (Twins-SVT's PEG, twins_svt.py:77-83) on the token map x[M, C] fp32 of B images of
 * gh x gw tokens, out of place:
 *   y[(b, i, j), c] = x[(b, i, j), c] + bias[c] + sum_{dy, dx < k} w[dy*k + dx][c] x[(b, i + dy - k/2, j + dx - k/2), c]
 * the depthwise k x k convolution with zero padding k / 2, plus the identity.  w fp32 [k*k][C] (tap major, channel
 * minor), bias fp32 [C]; y must not be x (every token reads its neighbours).  k = 1, 3, 5 or 7, C a multiple of 4;
 * x, w, bias and y 16-byte aligned.  Each image's output is computed from its own rows only.
 */
int b200vit_peg(const float* x, int64_t M, const float* w, const float* bias, float* y, int B, int gh, int gw, int C,
                int k, void* stream);

/*
 * CvT's convolutional projections, depthwise halves (DepthWiseConv2d up to its 1 x 1 convolution, cvt.py:51-60, 74-75),
 * on the LayerNorm'ed token map x[M, C] bf16 of B images of h x w tokens (token (b, y, x) at row (b*h + y)*w + x,
 * M = B*h*w), both outputs from one read of x:
 *   q_out[(b, y, x), c]  = bq[c]  + sum_{i, j < k} wq[i*k + j][c]  x[(b, y + i - k/2, x + j - k/2), c]
 *   kv_out[(b, r, q), c] = bkv[c] + sum_{i, j < k} wkv[i*k + j][c] x[(b, s*r + i - k/2, s*q + j - k/2), c]
 * q_out [M, C] bf16 (stride 1), kv_out [B*oh*ow, C] bf16 with oh = (h - 1)/s + 1, ow = (w - 1)/s + 1, row
 * (b*oh + r)*ow + q (stride s).  Taps outside the map are zero (padding k / 2).  wq, wkv fp32 [k*k][C] tap major and
 * bq, bkv fp32 [C], with the BatchNorm (eval) folded in by the caller: w * g / sqrt(var + eps), beta - mean * g /
 * sqrt(var + eps).  Sums in fp32 in tap order, rounded to bf16 once; no atomics, so repeated calls give the same bits.
 * k = 1, 3, 5 or 7, s >= 1, C a multiple of 8, B, h, w >= 1; all pointers 16-byte aligned; x overlaps neither output.
 * Each image's outputs come from its own rows only; nothing outside the B*h*w / B*oh*ow addressed rows is read or
 * written.
 */
int b200vit_conv_proj_dw(const void* x, int64_t M, const float* wq, const float* bq, const float* wkv,
                         const float* bkv, void* q_out, void* kv_out, int B, int h, int w, int C, int k, int s,
                         void* stream);

/*
 * CrossFormer's cross-scale embedding of the image (CrossEmbedLayer, crossformer.py:14-36) in one launch: S
 * convolutions of img [B, C, H, W] bf16 (NCHW, contiguous) with kernel sizes ks[0..S) and the one stride s, padding
 * p_i = (ks[i] - s) / 2, their outputs concatenated along the channels and written channels-last as fp32:
 *   out[(b*oh + r)*ow + q, off_i + n] = bias[off_i + n]
 *       + sum_{c, y, x < ks[i]} W_i[n, c, y, x] * img[b, c, r*s - p_i + y, q*s - p_i + x]
 * off_i = ns[0] + ... + ns[i-1], n < ns[i]; taps outside the image read zero.  Every scale must give the same oh x ow
 * map (the reference's torch.cat raises otherwise).  `w` holds the scales one after another, scale i as bf16
 * [ns[i], Kp_i] row-major with Kp_i = C*ks[i]^2 rounded up to a multiple of 64, columns (c, y, x) as in
 * Conv2d.weight.reshape(ns[i], -1), zeros past C*ks[i]^2; `bias` fp32 [sum ns] in output column order.  ks and ns are
 * host arrays.  An implicit GEMM on wgmma with fp32 accumulation: each CTA stages the input band of its output tokens
 * once in shared memory and gathers every scale's A k-blocks from it, so no im2col matrix is written.  Sums run in a
 * fixed order with no atomics, so repeated calls give the same bits.
 * 1 <= S <= B200VIT_CROSS_EMBED_MAX_SCALES, 1 <= C <= B200VIT_CROSS_EMBED_MAX_CHANNELS,
 * 1 <= s <= B200VIT_CROSS_EMBED_MAX_STRIDE, s <= ks[i] <= B200VIT_CROSS_EMBED_MAX_KERNEL, ns[i] a multiple of 8 up to
 * B200VIT_CROSS_EMBED_MAX_WIDTH; ldo even and >= sum ns; w 16-byte, out and bias 8-byte aligned.  Each image's outputs
 * come from its own pixels only; nothing outside the B*oh*ow addressed rows and their columns [0, sum ns) is written.
 */
int b200vit_cross_embed_nchw(const void* img, const void* w, const float* bias, float* out, int64_t ldo, int B, int C,
                             int H, int W, int S, const int* ks, const int* ns, int s, void* stream);

/*
 * ReLU then MaxPool2d(pk, stride ps, padding pp) in one pass (CCT's tokenizer, cct.py:187-190): y[M, C] bf16
 * channels-last (M = B*H*W, as b200vit_conv_im2col_nhwc's x) ->
 *   out[b*oh*ow + r*ow + q, c] = relu(max_{i, j < pk} y[(b, r*ps - pp + i, q*ps - pp + j), c]),
 * oh = (H + 2pp - pk) / ps + 1 (likewise ow), the padding counting as -inf; NaN propagates as in F.max_pool2d.
 * Exactly one output: out_bf16 (the next conv layer's channels-last input; ldo a multiple of 8) or out_f32 (the
 * tokens [B*oh*ow, C] b200vit_embed_tokens takes; ldo a multiple of 4), row stride ldo >= C elements.  C a multiple of
 * 8; 1 <= pk <= B200VIT_POOL_MAX_KERNEL, ps >= 1, 0 <= pp <= pk / 2, H + 2pp and W + 2pp >= pk; y and the output
 * 16-byte aligned.  Bit exact: every output is one of the inputs, or zero.
 */
int b200vit_relu_maxpool(const void* y, int64_t M, int B, int H, int W, int C, int pk, int ps, int pp, void* out_bf16,
                         float* out_f32, int64_t ldo, void* stream);

/*
 * Sequence pooling (CCT's TransformerClassifier with seq_pool, cct.py:284-288): x[B*n, D] fp32, token t of image b at
 * row b*n + t ->
 *   y_t = LayerNorm(x_t) (gamma, beta, eps),  z_t = y_t . w + bias[0],  out[b, :D] = sum_t softmax_t(z)_t y_t
 * as bf16 (the A operand of the classifier GEMM), row stride ldo.  fp32 throughout with an online max; each image's
 * tokens are shared by a cluster of up to 8 CTAs, merged in a fixed order (repeated calls give the same bits).  An
 * image's NaN or Inf reaches only its own output row.  D a multiple of 8 and <= B200VIT_SEQ_POOL_MAX_DIM, B <= 65535;
 * ldo a multiple of 8 and >= D; x, gamma, beta, w, out_bf16 16-byte aligned; bias a device pointer to one float.
 */
int b200vit_seq_pool(const float* x, int B, int n, int D, const float* gamma, const float* beta, float eps,
                     const float* w, const float* bias, void* out_bf16, int64_t ldo, void* stream);

/*
 * NesT's level boundaries (nest.py).  A level's stream is block-major: with its H x W map cut into nb x nb blocks of
 * sh x sw tokens (sh = H/nb, sw = W/nb), token (b, y, x) is at row
 *   ((b*nb + y/sh)*nb + x/sw)*(sh*sw) + (y % sh)*sw + (x % sw),
 * the reference's '(b b1 b2)' blocks with their tokens in '(h w)' order.  The last level (nb = 1) is in map order.
 *
 * b200vit_nest_level_entry: y[M, D] fp32 in map order (M = B*H*W, row (b*H + y)*W + x) ->
 *   x[block-major row of (b, r, q)] = max_{i, j < pk} LN(y[(b, r*ps - pp + i, q*ps - pp + j)]) + pos[(r % sh)*sw + q % sw]
 * over the oh x ow pooled map (oh = (H + 2pp - pk) / ps + 1, likewise ow) cut into nb x nb blocks of sh = oh/nb by
 * sw = ow/nb tokens.  LN is the LayerNorm over the D channels of a pixel (gamma, beta, eps; biased variance, eps
 * inside the sqrt); the pool counts padding as -inf and propagates NaN as F.max_pool2d does; pos[n_pos] fp32 is the
 * level's scalar position embedding, n_pos >= sh*sw.  xb_bf16 and stats (both or neither): the bf16 copy of x and its
 * row statistics [B*oh*ow][2], the bits b200vit_rowstats_cast writes for x.  1 <= pk <= B200VIT_NEST_POOL_MAX_KERNEL,
 * ps >= 1, 0 <= pp <= pk / 2, H + 2pp and W + 2pp >= pk, oh and ow multiples of nb; y, x, xb_bf16, gamma, beta
 * 16-byte aligned, stats 8-byte aligned; the outputs must not overlap y.  Exactly the B*oh*ow rows of x (xb_bf16,
 * stats) are written, and an output pixel reads only its own image's pool window.
 *
 * b200vit_nest_im2col: the A operand of a Conv2d(D, *, 3, padding = 1) over the map of a block-major stream x[M, D]
 * fp32 (M = B*H*W, nb x nb blocks) -> out[(b*H + y)*W + x, (i*3 + j)*D + c] bf16 = x[(b, y - 1 + i, x - 1 + j), c]
 * rounded to nearest, zero outside the map and in the K padding [9D, ldo).  D a multiple of 8, H and W multiples of
 * nb, ldo a multiple of 8 and >= 9D; x and out_bf16 16-byte aligned and not overlapping.
 */
#define B200VIT_NEST_POOL_MAX_KERNEL 3
int b200vit_nest_level_entry(const float* y, int64_t M, const float* gamma, const float* beta, float eps,
                             const float* pos, int n_pos, float* x, void* xb_bf16, float* stats, int B, int H, int W,
                             int D, int pk, int ps, int pp, int nb, void* stream);
int b200vit_nest_im2col(const float* x, int64_t M, void* out_bf16, int64_t ldo, int B, int H, int W, int D, int nb,
                        void* stream);

/*
 * ScalableViT's interactive windowed self-attention (scalable_vit.py:155-194) over B channels-last token maps:
 *   qkv[B*gh*gw, ld] bf16, token (b, y, x) at row (b*gh + y)*gw + x; columns q (H*dk) | k (H*dk) | v (H*dv),
 *   head-major.  The map is cut into wh x ww windows (wh = gh, ww = gw: the whole map); per window and head
 *     out = softmax(scale * q k^T) v + lim,
 *   lim[B*gh*gw, H*dv] bf16 the local interactive module's output in map order, out[B*gh*gw, H*dv] bf16 in map order
 *   (both contiguous).  The sum is formed in fp32, fma(O, 1 / l, lim) with O the unnormalised P V accumulator and l the
 *   softmax denominator, and rounded to bf16 once.
 * One CTA per 128 queries of a (window, head); keys and values stream in blocks of 64 with an fp32 online softmax,
 * both products on wgmma; rows are gathered from their map-order addresses by cp.async, rows past the window are
 * zero-filled and its keys masked.  One kernel for every window size from 1 to B200VIT_ATTN_KV_MAX_KEYS tokens.
 * gh and gw multiples of wh and ww; dk = 16, 32, 48 or 64 (a padded dim_key as for b200vit_attention_kv_ex); dv = 32
 * or 64; ld >= H*(2 dk + dv) and a multiple of 8; qkv, lim and out 16-byte aligned; out overlaps neither qkv nor lim;
 * H <= 65535.  Isolation: a window's output is computed from its own rows and its lim rows only, so a NaN or Inf stays
 * in its window, and nothing outside the B*gh*gw rows is read or written.
 */
int b200vit_attention_iwsa(const void* qkv, int64_t ld, const void* lim, void* out, int B, int gh, int gw, int wh,
                           int ww, int H, int dk, int dv, float scale, void* stream);

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
/* ... with rotary positions: b200vit_rope_qk(ws->qkv, rope_cs, rope_rows, ...) runs right after every layer's QKV GEMM
 * (vit_nd_rotary.py:137-147).  b200vit_encoder_blocks is this call with rope_cs = NULL. */
int b200vit_encoder_blocks_rope(const b200vit_layer* layers, int depth, float* x, const b200vit_encoder_ws* ws, int B,
                                int N, int D, int heads, int dh, int hidden, float scale, int primed,
                                const int32_t* cu_seqlens_dev, const int32_t* tile_prefix_dev, int total_tiles,
                                const float* rope_cs, int rope_rows, void* stream);
/* ... with a softmax scale per layer and attention flags: layer_scales is a HOST array of depth floats (NULL: `scale`
 * for every layer; LSA's learned temperature.exp(), vit_for_small_dataset.py:35,53), attn_flags goes to every
 * attention call (B200VIT_ATTN_MASK_SELF).  b200vit_encoder_blocks_rope is this call with (NULL, 0). */
int b200vit_encoder_blocks_ex(const b200vit_layer* layers, int depth, float* x, const b200vit_encoder_ws* ws, int B,
                              int N, int D, int heads, int dh, int hidden, float scale, int primed,
                              const int32_t* cu_seqlens_dev, const int32_t* tile_prefix_dev, int total_tiles,
                              const float* rope_cs, int rope_rows, const float* layer_scales, int attn_flags,
                              void* stream);

/*
 * T2T-ViT soft split (nn.Unfold(k, stride=s, padding=p) + Rearrange('b c n -> b n c'), t2t.py:37-38) as bit copies:
 *   out[b*oh*ow + r*ow + q, c*k*k + i*k + j] = src(b, c, r*s - p + i, q*s - p + j), 0 outside the map,
 * oh = (H + 2p - k) / s + 1 (likewise ow), channel-major columns (nn.Unfold's order), columns [C*k*k, ldo) zero filled.
 * Exactly one of out_bf16 (the A operand of a GEMM) and out_f32 (the fp32 residual stream of the soft-split Transformer
 * that follows) is given; ldo a multiple of 8 and >= C*k*k; out 16-byte aligned.  1 <= k, 1 <= s, 0 <= p < k, and the
 * padded map at least one window wide.  Every output row reads its own image's pixels / tokens only.
 * _image: src = img[B, C, H, W] bf16 (the first stage).
 * _tokens: src = x[B*n, ldx] bf16 (ldx >= C), the token rows of the previous soft-split Transformer's final LayerNorm,
 *   read as RearrangeImage does (t2t.py:20-22): a map of h = int(sqrt(n)) rows of w = n / h tokens, token r*w + c of
 *   image b at row b*n + r*w + c, channel c at column c.  An n that h does not divide is rejected (einops raises).
 */
int b200vit_t2t_unfold_image(const void* img, void* out_bf16, float* out_f32, int64_t ldo, int B, int C, int H, int W,
                             int k, int s, int p, void* stream);
int b200vit_t2t_unfold_tokens(const void* x, int64_t ldx, int B, int n, int C, void* out_bf16, float* out_f32,
                              int64_t ldo, int k, int s, int p, void* stream);

/*
 * Softmax attention of ONE head as wide as the token: the attention of a T2T-ViT soft-split Transformer (heads == 1,
 * dim_head == dim, t2t.py:40 / vit.py Attention), for widths past the 160 of b200vit_attention_varlen.
 *   qkv[B*n, 3*dp] bf16, columns [q | k | v], each padded from the true width w to dp with zero columns (zero rows of
 *   the projection), image b at rows b*n ..;  O = softmax(q k^T * scale) v, scale = w^-0.5 of the TRUE width.
 * The scores are materialised per image, in the caller's workspace (the library allocates nothing):
 *   S = scale * Q K^T in fp32 (wgmma: bf16 products, fp32 accumulation), P = softmax(S) rounded to bf16 once,
 *   O = P V accumulated in fp32 (wgmma) and rounded to bf16.
 * Outputs: out[B*n, dp] bf16 (may be NULL) and/or, x given, x[(b*n + i)*ldx + c] += bf16(O[b*n + i, c]) for
 * c < n_resid -- the residual add of the identity to_out (vit.py: heads == 1 and dim_head == dim) on the true columns.
 * Limits: n <= B200VIT_ATTN_WIDE_MAX_TOKENS, dp a multiple of 64 and <= B200VIT_ATTN_WIDE_MAX_WIDTH; qkv, out and ws
 * 16-byte aligned.  ws_bytes >= b200vit_attention_wide_workspace(n, dp, 1); the batch runs in chunks of as many images
 * as the workspace holds (b200vit_attention_wide_workspace(n, dp, images) bytes hold `images`), three launches each.
 * Isolation: q, k, v and P reach the tensor cores through 3-D tensor maps (column, token, image) that zero-fill past
 * each image's n tokens, so a NaN or Inf in one image leaves every other image's output bit-identical, and no row past
 * B*n is read.
 */
int64_t b200vit_attention_wide_workspace(int n, int dp, int images);
int b200vit_attention_wide(const void* qkv, void* out, float* x, int64_t ldx, int n_resid, int B, int n, int dp,
                           float scale, void* ws, int64_t ws_bytes, void* stream);

/*
 * Adaptive Token Sampling's token selection (ats_vit.py:48-109, 167-170) over images that each own a slot of S_in rows,
 * the first len_in[b] of them valid (row 0 the cls token):
 *   qkv[B*S_in, >= 3*H*dh] bf16 (row stride ld), packed [q | k | v] head-major as for b200vit_attention;
 *   len_in[B], ids_in[B*S_in]: DEVICE int32 valid lengths and the original token index of every row.
 * The layer samples iff max_b len_in[b] - 1 > K (the batch's padded length, so one image switches it for all).  Then,
 * per image, in fp32 over its valid rows only:
 *   p_h[j] = softmax_j(scale * q_h[0] . k_h[j]),  s_j = sum_h p_h[j] |v_h[j]| (j >= 1),
 *   l_c = log(s_{c+1} / (sum_j s_j + 1e-6) + 1e-6),  draw k: argmax_c (l_c - log(-log(u[b,k,c] + 1e-6) + 1e-6)), ties
 *   to the lowest c (torch.argmax), over c < len_in[b] - 1;
 * and row 0 plus the drawn rows 1 + c, once each in increasing order, are kept: U of them besides the cls row.
 *   u: [B, K, S_in - 1] uniforms in [0, 1], fp32 (u_bf16 = 0) or bf16 (u_bf16 = 1), contiguous; only c < len_in[b] - 1
 *   is read.
 * Outputs, S_out = min(S_in, K + 1) rows per image:
 *   src[B*S_out]: row r of image b comes from row src[b*S_out + r] = b*S_in + pos_r, pos_0 = 0, pos_1 < .. < pos_U the
 *     kept rows; rows r > U point at the cls row b*S_in (pad_sequence + F.pad, ats_vit.py:94-103);
 *   len_out[b] = 1 + U;  ids_out[b*S_out + r] = ids_in[b*S_in + pos_r].
 * Without sampling the map is the identity on the valid rows (pos_r = r for r < len_in[b], else 0) and
 * len_out = len_in.  len_out and ids_out must not be len_in and ids_in (every CTA reads all of len_in).
 * One CTA per image; S_in <= B200VIT_ATS_MAX_TOKENS, H * S_in <= B200VIT_ATS_MAX_HEAD_TOKENS, dh = 32, 64, 80 or 128,
 * ld a multiple of 8, qkv 16-byte aligned, B <= 65535.
 * Isolation: an image's selection reads only its own valid qkv rows and uniforms (and every image's len_in), so a NaN
 * or Inf in one image leaves every other image's outputs bit-identical.
 */
int b200vit_ats_select(const void* qkv, int64_t ld, const int32_t* len_in, const int32_t* ids_in, const void* u,
                       int u_bf16, int32_t* src, int32_t* len_out, int32_t* ids_out, int B, int S_in, int S_out, int K,
                       int H, int dh, float scale, void* stream);

/*
 * Row gather as bit copies (the residual stream and the kept queries after b200vit_ats_select, ats_vit.py:161-163):
 *   x_out[r, :D] = x[src[r], :D] (fp32, row strides ldx / ldx_out) when x is given;
 *   a_out[r, :ncols] = a[src[r], :ncols] (bf16, row strides lda / lda_out) when a is given; r < rows.
 * D, ldx, ldx_out multiples of 4; ncols, lda, lda_out multiples of 8; pointers 16-byte aligned; outputs distinct from
 * their inputs (other rows may still be read).
 */
int b200vit_ats_gather(const int32_t* src, int rows, const float* x, int64_t ldx, float* x_out, int64_t ldx_out, int D,
                       const void* a, int64_t lda, void* a_out, int64_t lda_out, int ncols, void* stream);

/*
 * TEST HOOKS -- process-global switches for A/B tests and bring-up; NOT part of the re-entrant API above (a value set
 * here changes every later call of every thread).  Production code never calls them.
 *   key 12: BLOCK_N of b200vit_gemm_bf16: 0 = auto (256 when N > 128, else 128; residual launches on the TMA-store
 *           epilogue: 128), 1 = 128, 2 = 256
 *   key 14: b200vit_gemm_bf16 epilogue: 0 = bf16 outputs and residual launches with ldo and N multiples of 8 are staged
 *           in shared memory and written by TMA stores (default; 256-wide residual tiles excepted), 1 = every launch
 *           stores straight from the accumulator registers.  Both give the same bits.
 *   key 15: b200vit_attention: 0 = launches with 128 < N <= 256 and dh = 32 or 64 run the persistent kernel (default),
 *           1 = every launch runs the tiled kernel.  Both give the same bits.
 */
int b200vit_debug_set(int key, int value);

#ifdef __cplusplus
}
#endif
#endif /* B200VIT_H_ */
