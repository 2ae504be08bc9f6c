// All encoder layers of a ViT in ONE call of the C ABI (reference vit.py:78-81: `for attn, ff in self.layers:
// x = attn(x) + x; x = ff(x) + x`), LayerNorm-folded schedule -- per layer five launches of this library's own kernels:
//   QKV GEMM (LN fold [+ per-head q/k RMSNorm])  ->  attention  ->  out-proj GEMM (+ residual, bf16 copy, row stats)
//   ->  FC1 GEMM (LN fold + bias + GELU)  ->  FC2 GEMM (+ bias + residual, bf16 copy, row stats).
// Nothing here touches the device itself: it is the host-side loop, moved below the language boundary so that a Python
// (ctypes) or C++ host pays one call instead of 5 x depth -- at small batches the forward is host bound.
// With a rope table (b200vit_encoder_blocks_rope) a sixth launch rotates q and k right after the QKV GEMM.
// b200vit_encoder_blocks_ex adds a softmax scale per layer and attention flags (LSA: learned temperature, self mask).
#include <cmath>

#include "../../include/b200vit.h"
#include "host_util.h"

using namespace b200;

// the ctypes mirror (vit_pytorch_b200/_lib.py: Layer, EncoderWs) is laid out by hand: pin the C side
static_assert(sizeof(b200vit_layer) == 11 * sizeof(void*) + 2 * sizeof(float), "b200vit_layer layout");
static_assert(sizeof(b200vit_encoder_ws) == 7 * sizeof(void*), "b200vit_encoder_ws layout");

extern "C" int b200vit_encoder_blocks(const b200vit_layer* layers, int depth, float* x, const b200vit_encoder_ws* ws,
                                      int B, int N, int D, int heads, int dh, int hidden, float scale, int primed,
                                      const int32_t* cu_seqlens_dev, const int32_t* tile_prefix_dev, int total_tiles,
                                      void* stream) {
  return b200vit_encoder_blocks_rope(layers, depth, x, ws, B, N, D, heads, dh, hidden, scale, primed, cu_seqlens_dev,
                                     tile_prefix_dev, total_tiles, nullptr, 0, stream);
}

extern "C" int b200vit_encoder_blocks_rope(const b200vit_layer* layers, int depth, float* x,
                                           const b200vit_encoder_ws* ws, int B, int N, int D, int heads, int dh,
                                           int hidden, float scale, int primed, const int32_t* cu_seqlens_dev,
                                           const int32_t* tile_prefix_dev, int total_tiles, const float* rope_cs,
                                           int rope_rows, void* stream) {
  return b200vit_encoder_blocks_ex(layers, depth, x, ws, B, N, D, heads, dh, hidden, scale, primed, cu_seqlens_dev,
                                   tile_prefix_dev, total_tiles, rope_cs, rope_rows, nullptr, 0, stream);
}

extern "C" int b200vit_encoder_blocks_ex(const b200vit_layer* layers, int depth, float* x,
                                         const b200vit_encoder_ws* ws, int B, int N, int D, int heads, int dh,
                                         int hidden, float scale, int primed, const int32_t* cu_seqlens_dev,
                                         const int32_t* tile_prefix_dev, int total_tiles, const float* rope_cs,
                                         int rope_rows, const float* layer_scales, int attn_flags, void* stream) {
  B200_CHECK_ARG(layers && x && ws && depth > 0, "encoder_blocks: null pointer / depth %d", depth);
  B200_CHECK_ARG(B > 0 && N > 0 && D > 0 && heads > 0 && hidden > 0, "encoder_blocks: bad shape");
  B200_CHECK_ARG(ws->xb && ws->qkv && ws->o && ws->h && ws->stats_in && ws->stats_a && ws->stats_b,
                 "encoder_blocks: incomplete workspace");
  B200_CHECK_ARG(N <= 512 || (cu_seqlens_dev && tile_prefix_dev && total_tiles > 0),
                 "encoder_blocks: N = %d > 512 needs the varlen index (cu_seqlens, tile_prefix)", N);
  B200_CHECK_ARG(!rope_cs || rope_rows > 0, "encoder_blocks: rope table with %d rows", rope_rows);
  B200_CHECK_ARG((attn_flags & ~B200VIT_ATTN_MASK_SELF) == 0, "encoder_blocks: unknown attention flags 0x%x",
                 attn_flags);
  if (layer_scales)
    for (int i = 0; i < depth; ++i)
      B200_CHECK_ARG(std::isfinite(layer_scales[i]), "encoder_blocks: layer %d has a non-finite scale", i);
  const int M = B * N, I = heads * dh;
  const int parts = b200vit_stats_parts(D);
  int rc = 0;
  if (!primed) {
    rc = b200vit_rowstats_cast(x, ws->xb, ws->stats_in, M, D, stream);
    if (rc) return rc;
  }
  for (int i = 0; i < depth; ++i) {
    const b200vit_layer& L = layers[i];
    B200_CHECK_ARG(L.qkv_wg && L.qkv_t && L.qkv_s && L.out_w && L.fc1_wg && L.fc1_t && L.fc1_s && L.fc2_w,
                   "encoder_blocks: layer %d has a null weight", i);
    const float* sums = i == 0 ? ws->stats_in : ws->stats_a;
    const int sum_parts = i == 0 ? 1 : parts;
    // x -> LN -> to_qkv   (vit.py:52-54; simple_vit_with_qk_norm.py:60-67 when qk_gamma is given)
    if (L.qk_gamma)
      rc = b200vit_gemm_headnorm_bf16(ws->xb, D, L.qkv_wg, D, ws->qkv, 3 * I, L.qkv_t, sums, sum_parts, L.ln1_eps,
                                      L.qkv_s, L.qk_gamma, 2 * heads, dh, 0.f, M, 3 * I, D,
                                      B200VIT_EPI_BIAS | B200VIT_EPI_LNFOLD, stream);
    else
      rc = b200vit_gemm_bf16(ws->xb, D, L.qkv_wg, D, ws->qkv, nullptr, 3 * I, L.qkv_t, nullptr, sums, sum_parts,
                             L.ln1_eps, L.qkv_s, nullptr, M, 3 * I, D, B200VIT_EPI_BIAS | B200VIT_EPI_LNFOLD, stream);
    if (rc) return rc;
    // rotary positions on q and k   (vit_nd_rotary.py:143-147)
    if (rope_cs) {
      rc = b200vit_rope_qk(ws->qkv, rope_cs, rope_rows, M, heads, dh, stream);
      if (rc) return rc;
    }
    // softmax(q k^T * scale) v, heads merged   (vit.py:55-63; vit_for_small_dataset.py:53-60 with the flags)
    const float sc = layer_scales ? layer_scales[i] : scale;
    if (N <= 512)
      rc = b200vit_attention_ex(ws->qkv, ws->o, B, N, heads, dh, sc, attn_flags, stream);
    else
      rc = b200vit_attention_varlen_ex(ws->qkv, ws->o, cu_seqlens_dev, tile_prefix_dev, B, M, total_tiles, heads, dh,
                                       sc, attn_flags, stream);
    if (rc) return rc;
    // to_out + residual   (vit.py:64,80)
    rc = b200vit_gemm_bf16(ws->o, I, L.out_w, I, ws->xb, x, D, L.out_b, x, nullptr, 0, 0.f, nullptr, ws->stats_b, M, D,
                           I, (L.out_b ? B200VIT_EPI_BIAS : 0) | B200VIT_EPI_RESIDUAL | B200VIT_EPI_STATS, stream);
    if (rc) return rc;
    // LN -> Linear -> GELU   (vit.py:19-21)
    rc = b200vit_gemm_bf16(ws->xb, D, L.fc1_wg, D, ws->h, nullptr, hidden, L.fc1_t, nullptr, ws->stats_b, parts,
                           L.ln2_eps, L.fc1_s, nullptr, M, hidden, D,
                           B200VIT_EPI_BIAS | B200VIT_EPI_GELU | B200VIT_EPI_LNFOLD, stream);
    if (rc) return rc;
    // Linear + residual   (vit.py:23,81)
    rc = b200vit_gemm_bf16(ws->h, hidden, L.fc2_w, hidden, ws->xb, x, D, L.fc2_b, x, nullptr, 0, 0.f, nullptr,
                           ws->stats_a, M, D, hidden,
                           (L.fc2_b ? B200VIT_EPI_BIAS : 0) | B200VIT_EPI_RESIDUAL | B200VIT_EPI_STATS, stream);
    if (rc) return rc;
  }
  return 0;
}
