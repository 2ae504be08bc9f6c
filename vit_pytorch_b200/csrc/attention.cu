// Multi-head softmax attention straight out of the packed QKV buffer, for sm_90a:
//   b200vit_attention          B sequences of N tokens (N <= 512)
//   b200vit_attention_varlen   packed sequences of any length (cu_seqlens), the block-diagonal attention of NaViT and
//                              the long-sequence path of ViT
// One CTA = one 128-row query tile of one (sequence, head): two warpgroups of 64 query rows each.  Thread 0 loads the
// Q tile and the K / V blocks of KB keys with TMA into a two-stage ring of 128B-swizzled shared memory (mbarrier
// complete_tx; a stage is reloaded once both warpgroups have released it).  Per key block each warpgroup computes
// S = Q K^T with wgmma (both operands in shared memory), runs an online softmax in fp32 on the accumulator registers
// and accumulates O += P V with wgmma, P (bf16) taken from registers as the A operand and V read as the transposed
// (MN-major) B operand.  dh = 64, or 80: an 80-wide head is a 64-wide (128B swizzle) plus a 16-wide (32B swizzle)
// slab.  Keys of a block beyond the sequence get probability 0; TMA zero-fills rows beyond the buffer.
#include "common.cuh"
#include "host_util.h"

namespace b200 {

constexpr int ATT_QROWS = 128;
constexpr int ATT_THREADS = 256;

struct AttnParams {
  __nv_bfloat16* out;
  int N;                      // fixed-length mode: tokens per sequence (grid.z = sequence)
  const int32_t* cu_seqlens;  // varlen mode: [num_seqs + 1] token offsets, tile_prefix: 128-row tiles before s
  const int32_t* tile_prefix;
  int num_seqs;
  int H, I;                   // heads, H * dh
  float scale_log2e;
};

template <int DH, int KB>
struct AttnSmem {
  static constexpr bool WIDE = DH == 80;
  static constexpr int Q64 = ATT_QROWS * 128;        // 64 columns, 128B swizzle
  static constexpr int Q16 = WIDE ? ATT_QROWS * 32 : 0;  // columns 64..79, 32B swizzle
  static constexpr int KV64 = KB * 128;
  static constexpr int KV16 = WIDE ? KB * 32 : 0;
  static constexpr int STAGE = 2 * (KV64 + KV16);   // K64 | V64 | K16 | V16
  static constexpr int STAGE_OFF = Q64 + Q16;
  static constexpr int BAR_OFF = STAGE_OFF + 2 * STAGE;
  static constexpr int BYTES = BAR_OFF + 5 * 8 + 1024;  // full[2], empty[2], q; slack for 1024B alignment
};

template <int DH, int KB, bool VARLEN, bool EMUL>
__global__ void __launch_bounds__(ATT_THREADS, (DH == 64 && KB == 64) ? 2 : 1)
attention_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmKV,
                 const __grid_constant__ CUtensorMap tmQ16, const __grid_constant__ CUtensorMap tmKV16,
                 const AttnParams p) {
  using L = AttnSmem<DH, KB>;
  constexpr bool WIDE = L::WIDE;
  constexpr int NS = KB / 2;  // score accumulators per thread
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + L::BAR_OFF);
  uint64_t* empty = full + 2;
  uint64_t* qbar = full + 4;

  const int h = blockIdx.y;
  int seq_start, len, q0;
  if (VARLEN) {
    const int tile = blockIdx.x;
    int lo = 0, hi = p.num_seqs - 1;  // last s with tile_prefix[s] <= tile
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (p.tile_prefix[mid] <= tile) lo = mid;
      else hi = mid - 1;
    }
    seq_start = p.cu_seqlens[lo];
    len = p.cu_seqlens[lo + 1] - seq_start;
    q0 = (tile - p.tile_prefix[lo]) * ATT_QROWS;
  } else {
    seq_start = blockIdx.z * p.N;
    len = p.N;
    q0 = blockIdx.x * ATT_QROWS;
  }
  const int nblocks = (len + KB - 1) / KB;
  const int colq = h * DH, colk = p.I + h * DH, colv = 2 * p.I + h * DH;
  const int tid = threadIdx.x;
  const int wg = tid >> 7, t = tid & 127, warp = t >> 5, lane = t & 31;

  auto issue_kv = [&](int blk) {
    const int st = blk & 1;
    uint8_t* sb = smem + L::STAGE_OFF + st * L::STAGE;
    const int row = seq_start + blk * KB;
    mbar_arrive_expect_tx(&full[st], L::STAGE);
    tma_load_2d(sb, &tmKV, &full[st], colk, row);
    tma_load_2d(sb + L::KV64, &tmKV, &full[st], colv, row);
    if (WIDE) {
      tma_load_2d(sb + 2 * L::KV64, &tmKV16, &full[st], colk + 64, row);
      tma_load_2d(sb + 2 * L::KV64 + L::KV16, &tmKV16, &full[st], colv + 64, row);
    }
  };

  if (tid == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmKV);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 2);  // one arrive per warpgroup
    }
    mbar_init(qbar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(qbar, L::Q64 + L::Q16);
    tma_load_2d(smem, &tmQ, qbar, colq, seq_start + q0);
    if (WIDE) tma_load_2d(smem + L::Q64, &tmQ16, qbar, colq + 64, seq_start + q0);
    issue_kv(0);
    if (nblocks > 1) issue_kv(1);
  }

  float o[32], o16[8];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) o16[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  const uint32_t qa = smem_u32(smem) + wg * 64 * 128;
  const uint32_t qa16 = smem_u32(smem + L::Q64) + wg * 64 * 32;
  mbar_wait(qbar, 0);

  for (int kb = 0; kb < nblocks; ++kb) {
    const int st = kb & 1;
    const uint32_t ph = (kb >> 1) & 1;
    mbar_wait(&full[st], ph);
    const uint32_t sb = smem_u32(smem + L::STAGE_OFF + st * L::STAGE);

    // S = Q K^T (64 rows x KB keys per warpgroup)
    float s[NS];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint64_t ad = make_wgmma_desc(qa, 1024, WGMMA_SW128) + 2 * k;
      const uint64_t bd = make_wgmma_desc(sb, 1024, WGMMA_SW128) + 2 * k;
      if constexpr (KB == 128) wgmma_m64n128k16(s, ad, bd, k != 0);
      else wgmma_m64n64k16(s, ad, bd, k != 0);
    }
    if constexpr (WIDE) {
      const uint64_t ad = make_wgmma_desc(qa16, 256, WGMMA_SW32);
      const uint64_t bd = make_wgmma_desc(sb + 2 * L::KV64, 256, WGMMA_SW32);
      if constexpr (KB == 128) wgmma_m64n128k16(s, ad, bd, 1);
      else wgmma_m64n64k16(s, ad, bd, 1);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(s);

    // online softmax (log2 units); s[4j + e]: row 16 warp + lane/4 + 8 (e >> 1), key 8 j + 2 (lane % 4) + (e & 1)
    const int key0 = kb * KB + 2 * (lane & 3);
    float mx[2] = {m[0], m[1]};
#pragma unroll
    for (int j = 0; j < KB / 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const bool valid = key0 + j * 8 + (e & 1) < len;
        s[4 * j + e] = valid ? s[4 * j + e] * p.scale_log2e : -INFINITY;
        mx[e >> 1] = fmaxf(mx[e >> 1], s[4 * j + e]);
      }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      const float corr = fast_ex2(m[r] - mx[r]);  // m = -inf on the first block: exp2(-inf) = 0
      l[r] *= corr;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        o[4 * i + 2 * r] *= corr;
        o[4 * i + 2 * r + 1] *= corr;
      }
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        o16[4 * i + 2 * r] *= corr;
        o16[4 * i + 2 * r + 1] *= corr;
      }
      m[r] = mx[r];
    }
#pragma unroll
    for (int j = 0; j < KB / 8; ++j) {
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        float e0, e1;
        const float x0 = s[4 * j + 2 * r] - m[r], x1 = s[4 * j + 2 * r + 1] - m[r];
        if (EMUL && (j & 1)) {
          // half of the exponentials on the FMA pipe (masked keys are -inf: forced to 0)
          exp2_emul2(f2_make(x0, x1), e0, e1);
          e0 = s[4 * j + 2 * r] == -INFINITY ? 0.f : e0;
          e1 = s[4 * j + 2 * r + 1] == -INFINITY ? 0.f : e1;
        } else {
          e0 = fast_ex2(x0);
          e1 = fast_ex2(x1);
        }
        s[4 * j + 2 * r] = e0;
        s[4 * j + 2 * r + 1] = e1;
        l[r] += e0 + e1;
      }
    }

    // O += P V: the score accumulators of 16 keys are the A fragment of one k-step (bf16)
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < KB / 16; ++kk) {
      const uint32_t a[4] = {pack_bf16x2(s[8 * kk], s[8 * kk + 1]), pack_bf16x2(s[8 * kk + 2], s[8 * kk + 3]),
                             pack_bf16x2(s[8 * kk + 4], s[8 * kk + 5]), pack_bf16x2(s[8 * kk + 6], s[8 * kk + 7])};
      wgmma_m64n64k16_rs_tb(o, a, make_wgmma_desc_lbo(sb + L::KV64 + kk * 2048, 1024, 1024, WGMMA_SW128));
      if constexpr (WIDE)
        wgmma_m64n16k16_rs_tb(o16, a, make_wgmma_desc_lbo(sb + 2 * L::KV64 + L::KV16 + kk * 512, 256, 256, WGMMA_SW32));
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(o);
    fence_regs(o16);
    if (t == 0) mbar_arrive(&empty[st]);
    if (tid == 0 && kb + 2 < nblocks) {
      mbar_wait(&empty[st], ph);  // both warpgroups are done with this stage
      issue_kv(kb + 2);
    }
  }

#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
    l[r] = 1.0f / l[r];
  }
  const int qr = q0 + wg * 64 + warp * 16 + (lane >> 2);
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = qr + 8 * r;
    if (row >= len) continue;
    __nv_bfloat16* op = p.out + (long long)(seq_start + row) * p.I + h * DH + 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < 8; ++j)
      *reinterpret_cast<uint32_t*>(op + j * 8) = pack_bf16x2(o[4 * j + 2 * r] * l[r], o[4 * j + 2 * r + 1] * l[r]);
    if constexpr (WIDE) {
#pragma unroll
      for (int j = 0; j < 2; ++j)
        *reinterpret_cast<uint32_t*>(op + 64 + j * 8) =
            pack_bf16x2(o16[4 * j + 2 * r] * l[r], o16[4 * j + 2 * r + 1] * l[r]);
    }
  }
}

// Tensor maps over qkv[T, 3 I]: 64-column boxes (128B swizzle) of 128 query rows / KB key rows, and -- dh 80 -- the
// same with 16 columns (32B swizzle).
template <int DH, int KB, bool VARLEN, bool EMUL>
static int launch_attention_t(const void* qkv, int T, const AttnParams& p, dim3 grid, cudaStream_t stream) {
  using L = AttnSmem<DH, KB>;
  CUtensorMap tm[4];
  const uint64_t dims[2] = {(uint64_t)3 * p.I, (uint64_t)T};
  const uint64_t strides[1] = {(uint64_t)3 * p.I * 2};
  const uint32_t qbox[2] = {64, ATT_QROWS}, kvbox[2] = {64, KB}, qbox16[2] = {16, ATT_QROWS}, kvbox16[2] = {16, KB};
  int rc = encode_tmap_bf16(&tm[0], qkv, 2, dims, strides, qbox);
  if (!rc) rc = encode_tmap_bf16(&tm[1], qkv, 2, dims, strides, kvbox);
  if (!rc && DH == 80) rc = encode_tmap_bf16_sw(&tm[2], qkv, 2, dims, strides, qbox16, 32);
  if (!rc && DH == 80) rc = encode_tmap_bf16_sw(&tm[3], qkv, 2, dims, strides, kvbox16, 32);
  if (rc) return rc;
  if (DH != 80) tm[2] = tm[0], tm[3] = tm[1];
  auto kern = attention_kernel<DH, KB, VARLEN, EMUL>;
  B200_ENSURE_SMEM(kern, L::BYTES);
  kern<<<grid, ATT_THREADS, L::BYTES, stream>>>(tm[0], tm[1], tm[2], tm[3], p);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

template <bool VARLEN>
static int launch_attention(const void* qkv, int T, const AttnParams& p, int dh, int kb, bool emul, dim3 grid,
                            cudaStream_t st) {
  if (dh == 80) {
    if (kb == 128) return emul ? launch_attention_t<80, 128, VARLEN, true>(qkv, T, p, grid, st)
                               : launch_attention_t<80, 128, VARLEN, false>(qkv, T, p, grid, st);
    return emul ? launch_attention_t<80, 64, VARLEN, true>(qkv, T, p, grid, st)
                : launch_attention_t<80, 64, VARLEN, false>(qkv, T, p, grid, st);
  }
  if (kb == 128) return emul ? launch_attention_t<64, 128, VARLEN, true>(qkv, T, p, grid, st)
                             : launch_attention_t<64, 128, VARLEN, false>(qkv, T, p, grid, st);
  return emul ? launch_attention_t<64, 64, VARLEN, true>(qkv, T, p, grid, st)
              : launch_attention_t<64, 64, VARLEN, false>(qkv, T, p, grid, st);
}

// test hooks (include/b200vit.h)
static std::atomic<int> g_attn_mode{0};    // key 1
static std::atomic<int> g_attn_emul{0};    // key 13
static std::atomic<int> g_varlen_mode{0};  // key 11

}  // namespace b200

using namespace b200;

extern "C" int b200vit_debug_set(int key, int value) {
  switch (key) {
    case 1: g_attn_mode = value; return 0;
    case 11: g_varlen_mode = value; return 0;
    case 12: gemm_set_block_n(value); return 0;
    case 13: g_attn_emul = value; return 0;
    default: return B200VIT_ERR_INVALID;
  }
}

extern "C" int b200vit_attention(const void* qkv, void* out, int B, int N, int H, int dh, float scale, void* stream) {
  B200_CHECK_ARG(qkv && out, "attention: null pointer");
  B200_CHECK_ARG(B > 0 && N > 0 && H > 0, "attention: bad shape B=%d N=%d H=%d", B, N, H);
  B200_CHECK_ARG(dh == 64 || dh == 80, "attention: dim_head=%d not supported by this build (64 or 80)", dh);
  B200_CHECK_ARG(N <= 512, "attention: N=%d > 512 goes through b200vit_attention_varlen", N);
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(qkv) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0,
                 "attention: pointers must be 16-byte aligned");
  B200_CHECK_ARG(B <= 65535, "attention: B=%d exceeds the grid", B);
  AttnParams p{};
  p.out = reinterpret_cast<__nv_bfloat16*>(out);
  p.N = N;
  p.H = H;
  p.I = H * dh;
  p.scale_log2e = scale * 1.4426950408889634f;
  const dim3 grid((N + ATT_QROWS - 1) / ATT_QROWS, H, B);
  return launch_attention<false>(qkv, B * N, p, dh, g_attn_mode.load() == 2 ? 128 : 64, g_attn_emul.load() != 0,
                                 grid, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int b200vit_attention_varlen(const void* qkv, void* out, const int32_t* cu_seqlens_dev,
                                        const int32_t* tile_prefix_dev, int num_seqs, int total_tokens, int total_tiles,
                                        int H, int dh, float scale, void* stream) {
  B200_CHECK_ARG(qkv && out && cu_seqlens_dev && tile_prefix_dev, "attention_varlen: null pointer");
  B200_CHECK_ARG(num_seqs > 0 && total_tokens > 0 && total_tiles > 0 && H > 0, "attention_varlen: bad shape");
  B200_CHECK_ARG(dh == 64 || dh == 80, "attention_varlen: dim_head=%d not supported by this build (64 or 80)", dh);
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(qkv) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0,
                 "attention_varlen: pointers must be 16-byte aligned");
  B200_CHECK_ARG(H <= 65535, "attention_varlen: H=%d exceeds the grid", H);
  AttnParams p{};
  p.out = reinterpret_cast<__nv_bfloat16*>(out);
  p.cu_seqlens = cu_seqlens_dev;
  p.tile_prefix = tile_prefix_dev;
  p.num_seqs = num_seqs;
  p.H = H;
  p.I = H * dh;
  p.scale_log2e = scale * 1.4426950408889634f;
  const int mode = g_varlen_mode.load();
  const dim3 grid(total_tiles, H, 1);
  return launch_attention<true>(qkv, total_tokens, p, dh, mode == 1 ? 128 : 64, mode == 2, grid,
                                reinterpret_cast<cudaStream_t>(stream));
}
