// Attention of LeViT (reference levit.py:40-108), for sm_90a: softmax attention with a learned per-head bias looked up
// from the 2-D offset between query and key, q / k heads of one width (dk) and v heads of another (dv), queries on a
// stride-s sub-grid of the keys' grid, and an optional GELU on the output.
//   b200vit_attention_posbias   out = [GELU] softmax_j(scale q.k + T[h][|dy| F + |dx|]) v
//
// One CTA = one warpgroup = 64 consecutive queries of one (image, head).  The queries are gathered from the full-grid
// qkv buffer: query n of the tile is the token (s i, s j), i = n / Fq, j = n % Fq, so the downsampling layer's q comes
// out of the same full-grid QKV GEMM as its keys and values.  Keys and values run in blocks of 64 through two shared-
// memory slots: every thread copies its 16-byte pieces with cp.async straight into the wgmma operand tiles of
// tile64.cuh, block kb + 1 in flight while block kb is computed.  Rows past the image's tokens are zero-filled without
// a read, so nothing outside the image is touched.
// The head's F*F bias values (times log2 e) are staged in shared memory once; each (query, key) index is formed from
// the coordinates in registers, so no [H, Nq, Nk] bias exists anywhere.  Per block: S = Q K^T with wgmma, the bias
// gathered and added, keys past Nk masked to -inf, the online softmax of attention.cu in fp32, O += P V with wgmma (P
// from registers, V as the transposed B operand).  Streaming every block (instead of keeping an image's keys
// resident) and the 64-query tile are untuned choices: no measurement preceded them.
#include "tile64.cuh"
#include "host_util.h"

namespace {

using namespace b200;
using namespace b200::tile64;

__device__ __forceinline__ float gelu_exact(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }

__device__ __forceinline__ uint32_t out_pair(float a, float b, float inv, bool gelu) {
  a *= inv;
  b *= inv;
  if (gelu) {
    a = gelu_exact(a);
    b = gelu_exact(b);
  }
  return pack_bf16x2(a, b);
}

struct PosBiasParams {
  const __nv_bfloat16* qkv;
  const float* table;      // [H][F*F]
  __nv_bfloat16* out;
  long long ld;
  int B, F, s, Fq, Nq, Nk, H;
  float scale_log2e;
  int gelu;
};

template <int DK, int DV>
__global__ void __launch_bounds__(THREADS)
attention_posbias_kernel(const PosBiasParams p) {
  using SK = Slabs<DK>;
  using SV = Slabs<DV>;
  constexpr int KV = SK::OP + SV::OP;  // one slot: K block | V block
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  // Q block, two K | V slots, then the head's bias table
  float* tab = reinterpret_cast<float*>(smem + SK::OP + 2 * KV);

  const int h = blockIdx.y, b = blockIdx.z;
  const int q0 = blockIdx.x * ROWS;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int F = p.F, Nk = p.Nk, nkb = (Nk + ROWS - 1) / ROWS;
  const long long img0 = (long long)b * Nk;  // first row of this image in qkv
  const uint32_t sq = smem_u32(smem), slot0 = sq + SK::OP;
  const int kcol = p.H * DK + h * DK, vcol = 2 * p.H * DK + h * DV;

  // queries: row n of the tile is the token (s i, s j) of the input grid
  load_block<DK>(sq, p.qkv, p.ld, h * DK, [&](int r) -> long long {
    const int n = q0 + r;
    if (n >= p.Nq) return -1;
    const int i = n / p.Fq, j = n - (n / p.Fq) * p.Fq;
    return img0 + (long long)(p.s * i) * F + p.s * j;
  }, tid);
  auto load_kv = [&](int kb) {
    const uint32_t base = slot0 + (kb & 1) * KV;
    auto key_row = [&](int r) -> long long {
      const int m = kb * ROWS + r;
      return m < Nk ? img0 + m : -1;
    };
    load_block<DK>(base, p.qkv, p.ld, kcol, key_row, tid);
    load_block<DV>(base + SK::OP, p.qkv, p.ld, vcol, key_row, tid);
  };
  load_kv(0);
  cp_async_commit();
  const float* th = p.table + (long long)h * Nk;
  for (int i = tid; i < Nk; i += THREADS) tab[i] = th[i] * 1.4426950408889634f;

  // this thread's two query rows r = 16 warp + lane/4 + 8 rh: their coordinates on the input grid
  int qy[2], qx[2];
#pragma unroll
  for (int rh = 0; rh < 2; ++rh) {
    const int n = min(q0 + warp * 16 + (lane >> 2) + 8 * rh, p.Nq - 1);  // rows past Nq: any valid position
    const int i = n / p.Fq;
    qy[rh] = p.s * i;
    qx[rh] = p.s * (n - i * p.Fq);
  }

  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  float o[SV::N64 > 0 ? SV::N64 : 1][32], o16[SV::N16 > 0 ? SV::N16 : 1][8];
#pragma unroll
  for (int c = 0; c < SV::N64; ++c)
#pragma unroll
    for (int i = 0; i < 32; ++i) o[c][i] = 0.f;
#pragma unroll
  for (int c = 0; c < SV::N16; ++c)
#pragma unroll
    for (int i = 0; i < 8; ++i) o16[c][i] = 0.f;

  for (int kb = 0; kb < nkb; ++kb) {
    // block kb + 1 goes into the other slot, which every thread finished reading at the end of block kb - 1
    if (kb + 1 < nkb) load_kv(kb + 1);
    cp_async_commit();
    cp_async_wait<1>();          // this thread's pieces of block kb (and of Q) have landed
    fence_proxy_async_smem();    // ... and are visible to wgmma
    __syncthreads();             // ... as are every other thread's, and the bias table

    const uint32_t sk = slot0 + (kb & 1) * KV, sv = sk + SK::OP;
    float s[32];
    wgmma_fence();
    qk_mma<DK>(s, sq, sk);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(s);

    // online softmax in log2 units; s[4 jj + e]: row half e >> 1, key 64 kb + 8 jj + 2 (lane % 4) + (e & 1)
    float mn[2] = {m[0], m[1]};
#pragma unroll
    for (int jj = 0; jj < 8; ++jj)
#pragma unroll
      for (int e1 = 0; e1 < 2; ++e1) {
        const int key = 64 * kb + 8 * jj + 2 * (lane & 3) + e1;
        const bool ok = key < Nk;
        const int ky = key / F, kx = key - (key / F) * F;
#pragma unroll
        for (int rh = 0; rh < 2; ++rh) {
          const int e = 2 * rh + e1;
          const int idx = abs(qy[rh] - ky) * F + abs(qx[rh] - kx);
          s[4 * jj + e] = ok ? fmaf(s[4 * jj + e], p.scale_log2e, tab[idx]) : -INFINITY;
          mn[rh] = fmaxf(mn[rh], s[4 * jj + e]);
        }
      }
    float alpha[2];
#pragma unroll
    for (int rh = 0; rh < 2; ++rh) {
      mn[rh] = fmaxf(mn[rh], __shfl_xor_sync(0xffffffffu, mn[rh], 1));
      mn[rh] = fmaxf(mn[rh], __shfl_xor_sync(0xffffffffu, mn[rh], 2));
      // every block holds at least one key, so mn is finite unless the scores are not
      alpha[rh] = fast_ex2(m[rh] - mn[rh]);
      m[rh] = mn[rh];
      l[rh] *= alpha[rh];
    }
#pragma unroll
    for (int jj = 0; jj < 8; ++jj)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int rh = e >> 1;
        const float v = fast_ex2(s[4 * jj + e] - m[rh]);
        s[4 * jj + e] = v;
        l[rh] += v;  // this thread's keys only: summed over the four lanes of the row after the last block
      }
#pragma unroll
    for (int c = 0; c < SV::N64; ++c)
#pragma unroll
      for (int i = 0; i < 32; ++i) o[c][i] *= alpha[(i >> 1) & 1];
#pragma unroll
    for (int c = 0; c < SV::N16; ++c)
#pragma unroll
      for (int i = 0; i < 8; ++i) o16[c][i] *= alpha[(i >> 1) & 1];
#pragma unroll
    for (int c = 0; c < SV::N64; ++c) fence_regs(o[c]);
#pragma unroll
    for (int c = 0; c < SV::N16; ++c) fence_regs(o16[c]);
    wgmma_fence();
    pv_mma<DV>(o, o16, s, sv);
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int c = 0; c < SV::N64; ++c) fence_regs(o[c]);
#pragma unroll
    for (int c = 0; c < SV::N16; ++c) fence_regs(o16[c]);
    __syncthreads();  // every thread is done with this slot: the next iteration refills it
  }

  const int I = p.H * DV;
  const bool gelu = p.gelu != 0;
#pragma unroll
  for (int rh = 0; rh < 2; ++rh) {
    l[rh] += __shfl_xor_sync(0xffffffffu, l[rh], 1);
    l[rh] += __shfl_xor_sync(0xffffffffu, l[rh], 2);
    const int n = q0 + warp * 16 + (lane >> 2) + 8 * rh;
    if (n >= p.Nq) continue;
    const float inv = 1.0f / l[rh];
    __nv_bfloat16* op = p.out + ((long long)b * p.Nq + n) * I + h * DV + 2 * (lane & 3);
#pragma unroll
    for (int c = 0; c < SV::N64; ++c)
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
        *reinterpret_cast<uint32_t*>(op + 64 * c + jj * 8) =
            out_pair(o[c][4 * jj + 2 * rh], o[c][4 * jj + 2 * rh + 1], inv, gelu);
#pragma unroll
    for (int c = 0; c < SV::N16; ++c)
#pragma unroll
      for (int jj = 0; jj < 2; ++jj)
        *reinterpret_cast<uint32_t*>(op + 64 * SV::N64 + 16 * c + jj * 8) =
            out_pair(o16[c][4 * jj + 2 * rh], o16[c][4 * jj + 2 * rh + 1], inv, gelu);
  }
}

template <int DK, int DV>
int launch_posbias(const PosBiasParams& p, cudaStream_t stream) {
  constexpr int KV = Slabs<DK>::OP + Slabs<DV>::OP;
  const int bytes = Slabs<DK>::OP + 2 * KV + B200VIT_ATTN_POSBIAS_MAX_KEYS * 4 + 1024;  // slack for 1024B alignment
  auto kern = attention_posbias_kernel<DK, DV>;
  B200_ENSURE_SMEM(kern, bytes);
  kern<<<dim3((p.Nq + ROWS - 1) / ROWS, p.H, p.B), THREADS, bytes, stream>>>(p);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

template <int DK>
int launch_dv(const PosBiasParams& p, int dv, cudaStream_t st) {
  switch (dv) {
    case 32: return launch_posbias<DK, 32>(p, st);
    case 64: return launch_posbias<DK, 64>(p, st);
    default: return launch_posbias<DK, 128>(p, st);
  }
}

}  // namespace

static inline bool aligned16(const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; }

extern "C" int b200vit_attention_posbias(const void* qkv, int64_t ld, void* out, const float* table, int B, int F,
                                         int s, int H, int dk, int dv, float scale, int flags, void* stream) {
  B200_CHECK_ARG(qkv && out && table, "attention_posbias: null pointer");
  B200_CHECK_ARG(B > 0 && F > 0 && H > 0, "attention_posbias: bad shape B=%d F=%d H=%d", B, F, H);
  B200_CHECK_ARG(s == 1 || s == 2, "attention_posbias: query stride s=%d (1 or 2)", s);
  B200_CHECK_ARG(dk == 16 || dk == 32 || dk == 64, "attention_posbias: dim_key=%d not built (16, 32 or 64)", dk);
  B200_CHECK_ARG(dv == 32 || dv == 64 || dv == 128, "attention_posbias: dim_value=%d not built (32, 64 or 128)", dv);
  B200_CHECK_ARG((long long)F * F <= B200VIT_ATTN_POSBIAS_MAX_KEYS, "attention_posbias: F=%d, %lld keys > %d", F,
                 (long long)F * F, B200VIT_ATTN_POSBIAS_MAX_KEYS);
  B200_CHECK_ARG(ld >= (int64_t)H * (2 * dk + dv) && ld % 8 == 0,
                 "attention_posbias: ld=%lld must be a multiple of 8 and >= %d", (long long)ld, H * (2 * dk + dv));
  B200_CHECK_ARG((flags & ~B200VIT_ATTN_GELU_OUT) == 0, "attention_posbias: unknown flags 0x%x", flags);
  B200_CHECK_ARG(aligned16(qkv) && aligned16(out) && aligned16(table),
                 "attention_posbias: pointers must be 16-byte aligned");
  B200_CHECK_ARG(H <= 65535 && B <= 65535, "attention_posbias: B=%d, H=%d exceed the grid", B, H);
  PosBiasParams p{};
  p.qkv = reinterpret_cast<const __nv_bfloat16*>(qkv);
  p.table = table;
  p.out = reinterpret_cast<__nv_bfloat16*>(out);
  p.ld = ld;
  p.B = B;
  p.F = F;
  p.s = s;
  p.Fq = (F + s - 1) / s;
  p.Nq = p.Fq * p.Fq;
  p.Nk = F * F;
  p.H = H;
  p.scale_log2e = scale * 1.4426950408889634f;
  p.gelu = (flags & B200VIT_ATTN_GELU_OUT) != 0;
  const auto st = reinterpret_cast<cudaStream_t>(stream);
  switch (dk) {
    case 16: return launch_dv<16>(p, dv, st);
    case 32: return launch_dv<32>(p, dv, st);
    default: return launch_dv<64>(p, dv, st);
  }
}
