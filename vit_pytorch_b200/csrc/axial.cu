// Softmax attention over short strided sequences straight out of the packed QKV buffer, for sm_90a:
//   b200vit_attention_axial   ViViT's attention along the time axis (reference vivit.py:144-150) and the masked
//                             temporal transformer (vivit.py:268), with an optional per-sequence key mask
// Tokens are [B][L][G] rows: token j of sequence s = b*G + p is row b*L*G + j*G + p of qkv[T, 3*H*dh] and of out.
// One CTA = one warpgroup = one 64-row tile of one head that holds SP whole sequences (SP adjacent p of one b, all L
// tokens of each).  Thread 0 loads Q, K and V with one TMA box per slab over the 4-D view (column, p, j, b) of qkv: box
// row r = j * SP + ip; out-of-range p are zero-filled.  A tile never holds two batch elements: O = P V meets every V
// row of the tile, and a masked key's zero probability times a NaN or Inf value would carry one video's non-finite
// input into another's output.  S = Q K^T (64 x 64) with wgmma, then a
// block-diagonal mask (same sequence) and the key mask in registers and a plain softmax in fp32 (every key of a row is
// in the tile), and O = P V with wgmma, P (bf16) taken from registers as the A operand and V read as the transposed
// (MN-major) B operand, as in attention.cu.  dh = 32, 64, 80 or 128 in 64-wide (128B swizzle) and 16-wide (32B swizzle)
// slabs.  A query row whose keys are all masked gets 0 (zero_masked_rows, scaled_dot_product_attention's result) or
// the mean of the L values of its sequence (masked_fill(-finfo.max) before the softmax, vivit.py:91-94).
#include "common.cuh"
#include "host_util.h"

namespace b200 {

constexpr int AX_ROWS = 64;
constexpr int AX_THREADS = 128;

struct AxialParams {
  __nv_bfloat16* out;
  const uint8_t* key_mask;  // NULL, or [B][L] with 1 = keep
  int B, L, G, I;           // I = H * dh
  int sp, tiles_p;          // sequences per tile along p; tiles along p
  float scale_log2e;
  int zero_masked_rows;
};

// Shared memory: Q | K | V, each N64 slabs 64 columns wide followed by N16 slabs 16 columns wide, 64 rows per slab.
template <int DH>
struct AxialSmem {
  static constexpr int N64 = DH / 64;
  static constexpr int N16 = (DH % 64) / 16;
  static_assert(N64 * 64 + N16 * 16 == DH, "dim_head must be a multiple of 16");
  static constexpr int S64 = AX_ROWS * 128;
  static constexpr int S16 = AX_ROWS * 32;
  static constexpr int OP = N64 * S64 + N16 * S16;  // one operand (q, k or v)
  static constexpr int BAR_OFF = 3 * OP;
  static constexpr int BYTES = BAR_OFF + 8 + 1024;  // barrier; slack for 1024B alignment
};

template <int DH>
__global__ void __launch_bounds__(AX_THREADS)
attention_axial_kernel(const __grid_constant__ CUtensorMap tm64, const __grid_constant__ CUtensorMap tm16,
                       const AxialParams p) {
  using S = AxialSmem<DH>;
  constexpr int N64 = S::N64, N16 = S::N16;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + S::BAR_OFF);

  const int h = blockIdx.y;
  const int tp = blockIdx.x % p.tiles_p, b0 = blockIdx.x / p.tiles_p;
  const int p0 = tp * p.sp;
  const int rows = p.sp * p.L;  // rows the box covers (<= 64)
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  // rows beyond the box: their keys are masked, but V meets a zero probability in O = P V and must be finite
  const uint4 z = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
  for (int o = 0; o < 3; ++o) {
#pragma unroll
    for (int c = 0; c < N64; ++c) {
      uint4* sl = reinterpret_cast<uint4*>(smem + o * S::OP + c * S::S64);
      for (int i = rows * 8 + tid; i < AX_ROWS * 8; i += AX_THREADS) sl[i] = z;
    }
#pragma unroll
    for (int c = 0; c < N16; ++c) {
      uint4* sl = reinterpret_cast<uint4*>(smem + o * S::OP + N64 * S::S64 + c * S::S16);
      for (int i = rows * 2 + tid; i < AX_ROWS * 2; i += AX_THREADS) sl[i] = z;
    }
  }
  fence_proxy_async_smem();
  if (tid == 0) {
    tma_prefetch_desc(&tm64);
    mbar_init(bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(bar, 3 * rows * DH * 2);  // zero-filled elements count too
#pragma unroll
    for (int o = 0; o < 3; ++o) {
      const int col = o * p.I + h * DH;
#pragma unroll
      for (int c = 0; c < N64; ++c) tma_load_4d(smem + o * S::OP + c * S::S64, &tm64, bar, col + 64 * c, p0, 0, b0);
#pragma unroll
      for (int c = 0; c < N16; ++c)
        tma_load_4d(smem + o * S::OP + N64 * S::S64 + c * S::S16, &tm16, bar, col + 64 * N64 + 16 * c, p0, 0, b0);
    }
  }

  // this thread's rows r = 16 warp + lane/4 + 8 rh and key columns c = 8 jj + 2 (lane % 4) + e1 (wgmma m64 layout):
  // sequence within the tile, and whether the key is in range and kept by the mask
  int rseq[2];
#pragma unroll
  for (int rh = 0; rh < 2; ++rh) rseq[rh] = (warp * 16 + (lane >> 2) + 8 * rh) % p.sp;
  int cseq[16];
  uint32_t kept = 0;
#pragma unroll
  for (int ci = 0; ci < 16; ++ci) {
    const int c = 8 * (ci >> 1) + 2 * (lane & 3) + (ci & 1);
    const int ip = c % p.sp, j = c / p.sp;
    cseq[ci] = c < rows ? ip : -1;  // columns beyond the box belong to no sequence (an all-masked row averages its own)
    bool ok = c < rows && p0 + ip < p.G;
    if (ok && p.key_mask) ok = p.key_mask[(long long)b0 * p.L + j] != 0;
    kept |= (ok ? 1u : 0u) << ci;
  }

  mbar_wait(bar, 0);

  // S = Q K^T: one k16 step per 16 columns, the 64-wide slabs first
  float s[32];
  const uint32_t sq = smem_u32(smem), sk = sq + S::OP, sv = sq + 2 * S::OP;
  wgmma_fence();
#pragma unroll
  for (int c = 0; c < N64; ++c)
#pragma unroll
    for (int k = 0; k < 4; ++k)
      wgmma_m64n64k16(s, make_wgmma_desc(sq + c * S::S64, 1024, WGMMA_SW128) + 2 * k,
                      make_wgmma_desc(sk + c * S::S64, 1024, WGMMA_SW128) + 2 * k, c != 0 || k != 0);
#pragma unroll
  for (int c = 0; c < N16; ++c)
    wgmma_m64n64k16(s, make_wgmma_desc(sq + N64 * S::S64 + c * S::S16, 256, WGMMA_SW32),
                    make_wgmma_desc(sk + N64 * S::S64 + c * S::S16, 256, WGMMA_SW32), N64 != 0 || c != 0);
  wgmma_commit();
  wgmma_wait<0>();
  fence_regs(s);

  // plain softmax in log2 units; s[4 jj + e]: row half e >> 1, key column index ci = 2 jj + (e & 1)
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int jj = 0; jj < 8; ++jj)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int ci = 2 * jj + (e & 1), rh = e >> 1;
      const bool ok = ((kept >> ci) & 1u) && cseq[ci] == rseq[rh];
      s[4 * jj + e] = ok ? s[4 * jj + e] * p.scale_log2e : -INFINITY;
      mx[rh] = fmaxf(mx[rh], s[4 * jj + e]);
    }
  float l[2];
#pragma unroll
  for (int rh = 0; rh < 2; ++rh) {
    mx[rh] = fmaxf(mx[rh], __shfl_xor_sync(0xffffffffu, mx[rh], 1));
    mx[rh] = fmaxf(mx[rh], __shfl_xor_sync(0xffffffffu, mx[rh], 2));
    l[rh] = 0.f;
  }
#pragma unroll
  for (int jj = 0; jj < 8; ++jj)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int ci = 2 * jj + (e & 1), rh = e >> 1;
      float v;
      if (mx[rh] != -INFINITY) v = fast_ex2(s[4 * jj + e] - mx[rh]);  // masked keys: exp2(-inf) = 0
      else v = (!p.zero_masked_rows && cseq[ci] == rseq[rh]) ? 1.f : 0.f;  // no key kept
      s[4 * jj + e] = v;
      l[rh] += v;
    }
#pragma unroll
  for (int rh = 0; rh < 2; ++rh) {
    l[rh] += __shfl_xor_sync(0xffffffffu, l[rh], 1);
    l[rh] += __shfl_xor_sync(0xffffffffu, l[rh], 2);
    l[rh] = l[rh] > 0.f ? 1.0f / l[rh] : 0.f;
  }

  // O = P V: the probabilities of 16 keys are the A fragment of one k-step (bf16); one MMA per slab
  float o[N64 > 0 ? N64 : 1][32], o16[N16 > 0 ? N16 : 1][8];
#pragma unroll
  for (int c = 0; c < N64; ++c)
#pragma unroll
    for (int i = 0; i < 32; ++i) o[c][i] = 0.f;
#pragma unroll
  for (int c = 0; c < N16; ++c)
#pragma unroll
    for (int i = 0; i < 8; ++i) o16[c][i] = 0.f;
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    const uint32_t a[4] = {pack_bf16x2(s[8 * kk], s[8 * kk + 1]), pack_bf16x2(s[8 * kk + 2], s[8 * kk + 3]),
                           pack_bf16x2(s[8 * kk + 4], s[8 * kk + 5]), pack_bf16x2(s[8 * kk + 6], s[8 * kk + 7])};
#pragma unroll
    for (int c = 0; c < N64; ++c)
      wgmma_m64n64k16_rs_tb(o[c], a, make_wgmma_desc_lbo(sv + c * S::S64 + kk * 2048, 1024, 1024, WGMMA_SW128));
#pragma unroll
    for (int c = 0; c < N16; ++c)
      wgmma_m64n16k16_rs_tb(o16[c], a,
                            make_wgmma_desc_lbo(sv + N64 * S::S64 + c * S::S16 + kk * 512, 256, 256, WGMMA_SW32));
  }
  wgmma_commit();
  wgmma_wait<0>();
#pragma unroll
  for (int c = 0; c < N64; ++c) fence_regs(o[c]);
#pragma unroll
  for (int c = 0; c < N16; ++c) fence_regs(o16[c]);

#pragma unroll
  for (int rh = 0; rh < 2; ++rh) {
    const int r = warp * 16 + (lane >> 2) + 8 * rh;
    const int ip = r % p.sp, j = r / p.sp, pp = p0 + ip;
    if (r >= rows || pp >= p.G) continue;
    __nv_bfloat16* op = p.out + (((long long)b0 * p.L + j) * p.G + pp) * p.I + h * DH + 2 * (lane & 3);
#pragma unroll
    for (int c = 0; c < N64; ++c)
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
        *reinterpret_cast<uint32_t*>(op + 64 * c + jj * 8) =
            pack_bf16x2(o[c][4 * jj + 2 * rh] * l[rh], o[c][4 * jj + 2 * rh + 1] * l[rh]);
#pragma unroll
    for (int c = 0; c < N16; ++c)
#pragma unroll
      for (int jj = 0; jj < 2; ++jj)
        *reinterpret_cast<uint32_t*>(op + 64 * N64 + 16 * c + jj * 8) =
            pack_bf16x2(o16[c][4 * jj + 2 * rh] * l[rh], o16[c][4 * jj + 2 * rh + 1] * l[rh]);
  }
}

// Tensor maps over the 4-D view (column, p, j, b) of qkv: boxes of 64 columns (128B swizzle) and 16 columns (32B
// swizzle) by SP x L x 1 tokens.  A kind the head does not use gets a copy of the other (never read).
template <int DH>
static int launch_axial_t(const void* qkv, const AxialParams& p, int H, int tiles, cudaStream_t stream) {
  using S = AxialSmem<DH>;
  CUtensorMap tm[2];
  const uint64_t ld = (uint64_t)3 * p.I;
  const uint64_t dims[4] = {ld, (uint64_t)p.G, (uint64_t)p.L, (uint64_t)p.B};
  const uint64_t strides[3] = {ld * 2, ld * 2 * p.G, ld * 2 * p.G * p.L};
  const uint32_t box64[4] = {64, (uint32_t)p.sp, (uint32_t)p.L, 1};
  const uint32_t box16[4] = {16, (uint32_t)p.sp, (uint32_t)p.L, 1};
  int rc = 0;
  if (S::N64) rc = encode_tmap_bf16(&tm[0], qkv, 4, dims, strides, box64);
  if (!rc && S::N16) rc = encode_tmap_bf16_sw(&tm[1], qkv, 4, dims, strides, box16, 32);
  if (rc) return rc;
  if (!S::N16) tm[1] = tm[0];
  if (!S::N64) tm[0] = tm[1];
  auto kern = attention_axial_kernel<DH>;
  B200_ENSURE_SMEM(kern, S::BYTES);
  kern<<<dim3(tiles, H), AX_THREADS, S::BYTES, stream>>>(tm[0], tm[1], p);
  B200_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

}  // namespace b200

using namespace b200;

extern "C" int b200vit_attention_axial(const void* qkv, void* out, const uint8_t* key_mask, int B, int L, int G, int H,
                                       int dh, float scale, int zero_masked_rows, void* stream) {
  B200_CHECK_ARG(qkv && out, "attention_axial: null pointer");
  B200_CHECK_ARG(B > 0 && L > 0 && G > 0 && H > 0, "attention_axial: bad shape B=%d L=%d G=%d H=%d", B, L, G, H);
  B200_CHECK_ARG(head_width_ok(dh), "attention_axial: dim_head=%d not supported by this build (32, 64, 80 or 128)",
                 dh);
  B200_CHECK_ARG(L <= AX_ROWS, "attention_axial: L=%d > %d (a sequence must fit one 64-row tile)", L, AX_ROWS);
  B200_CHECK_ARG((reinterpret_cast<uintptr_t>(qkv) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0,
                 "attention_axial: pointers must be 16-byte aligned");
  B200_CHECK_ARG(H <= 65535, "attention_axial: H=%d exceeds the grid", H);
  AxialParams p{};
  p.out = reinterpret_cast<__nv_bfloat16*>(out);
  p.key_mask = key_mask;
  p.B = B;
  p.L = L;
  p.G = G;
  p.I = H * dh;
  p.sp = G < AX_ROWS / L ? G : AX_ROWS / L;
  p.tiles_p = (G + p.sp - 1) / p.sp;
  const long long tiles = (long long)p.tiles_p * B;
  B200_CHECK_ARG(tiles <= 0x7fffffffLL, "attention_axial: %lld tiles exceed the grid", tiles);
  p.scale_log2e = scale * 1.4426950408889634f;
  p.zero_masked_rows = zero_masked_rows != 0;
  const auto st = reinterpret_cast<cudaStream_t>(stream);
  switch (dh) {
    case 32: return launch_axial_t<32>(qkv, p, H, (int)tiles, st);
    case 80: return launch_axial_t<80>(qkv, p, H, (int)tiles, st);
    case 128: return launch_axial_t<128>(qkv, p, H, (int)tiles, st);
    default: return launch_axial_t<64>(qkv, p, H, (int)tiles, st);
  }
}
