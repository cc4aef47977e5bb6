// Global multi-head attention forward on wgmma (flash-attention, d = 64, no mask), sm_90a.
//
// One CTA = one (clip, head) and one 128-query tile, two warpgroups of 64 queries that share the K/V stream:
//   warp 8      TMA producer: the Q tile once, then K_j / V_j tiles (128 keys x 64, 128B swizzle) through a 3-deep ring
//   warps 0..7  warpgroup h owns query rows [64h, 64h + 64): S = Q K_j^T (wgmma 64 x 128 x 16, fp32 in registers),
//               one pass over S per key tile — p = 2^(s*c - m_ref) against a reference exponent m_ref that is the row
//               maximum of the first tile and is only raised (by a whole power of two, so the rescale of O and L is
//               exact) when a later tile produces p > 2^8 —, P packed to bf16 in registers as the A operand of
//               O += P V_j (wgmma 64 x 64 x 16, V consumed MN-major straight from its TMA tile), and the denominator L
//               summed over exactly the bf16 P that the numerator uses.  Each row's 128 scores of a tile live in the
//               four lanes of a quad; row maxima and sums combine by shuffles.
#include <cudaTypedefs.h>

#include "common.cuh"
#include "tmap.cuh"
#include "ptx.cuh"

namespace pgt {

constexpr int FT_D = 64;
constexpr int FT_BM = 128;                 // queries per CTA (64 per warpgroup)
constexpr int FT_BN = 128;                 // keys per tile
constexpr int FT_NST = 3;                  // K/V ring depth
constexpr int FT_TILE = FT_BN * FT_D * 2;  // 16 KB: one 128 x 64 bf16 tile
constexpr int FT_THREADS = 256 + 32;
constexpr int FT_SMEM = FT_TILE /*Q*/ + FT_NST * 2 * FT_TILE /*K,V*/ + 256 + 1024;
constexpr float FT_TAU = 256.f;              // p above this raises the reference exponent for the following tiles

__global__ void __launch_bounds__(FT_THREADS, 1)
mha_tc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
              const __grid_constant__ CUtensorMap tmV, int L, __nv_bfloat16* __restrict__ out, int ldo) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;                                   // [16 KB]
  uint8_t* sK = sQ + FT_TILE;                           // [NST][16 KB]
  uint8_t* sV = sK + FT_NST * FT_TILE;                  // [NST][16 KB]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + FT_NST * FT_TILE);
  uint64_t* q_full = bars;                              // [1]
  uint64_t* kv_full = bars + 1;                         // [NST]
  uint64_t* kv_empty = kv_full + FT_NST;                // [NST] one arrive per consumer warp

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = blockIdx.y, clip = blockIdx.z;
  const int q0 = clip * L + blockIdx.x * FT_BM;         // first query row (global token index) of this CTA
  const int kv0 = clip * L;
  const int NT = L / FT_BN;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV);
    mbar_init(q_full, 1);
    for (int i = 0; i < FT_NST; ++i) { mbar_init(&kv_full[i], 1); mbar_init(&kv_empty[i], 8); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ------------------------------------------------------------------ TMA producer
    if (elect_one()) {
      mbar_arrive_expect_tx(q_full, FT_TILE);
      tma_load_2d(sQ, &tmQ, q_full, h * FT_D, q0);
    }
    __syncwarp();
    int st = 0;
    uint32_t ph = 0;
    for (int j = 0; j < NT; ++j) {
      mbar_wait(&kv_empty[st], ph ^ 1);
      if (elect_one()) {
        mbar_arrive_expect_tx(&kv_full[st], 2 * FT_TILE);
        tma_load_2d(sK + st * FT_TILE, &tmK, &kv_full[st], h * FT_D, kv0 + j * FT_BN);
        tma_load_2d(sV + st * FT_TILE, &tmV, &kv_full[st], h * FT_D, kv0 + j * FT_BN);
      }
      __syncwarp();
      if (++st == FT_NST) { st = 0; ph ^= 1; }
    }
  } else {
    // ------------------------------------------------------------------ attention warpgroups
    const int wg = warp >> 2, w = warp & 3;
    const int t4 = lane & 3;
    const float sl2 = 0.125f * 1.4426950408889634f;     // d^-1/2 * log2(e)
    const uint64_t dq = wgmma_desc_k_sw128(smem_u32(sQ) + wg * 64 * 128);
    float o[FT_D / 2];                                   // O: rows (g, g + 8) of the warp's 16, 64 columns
    float mb[2] = {0.f, 0.f};                            // reference exponent per row (log2 domain)
    float lsum[2] = {0.f, 0.f};                          // this lane's share of the row sums of the bf16 P
    int pending[2] = {0, 0};                             // raise the reference by 2^pending before the next tile
#pragma unroll
    for (int i = 0; i < FT_D / 2; ++i) o[i] = 0.f;
    mbar_wait(q_full, 0);
    int st = 0;
    uint32_t ph = 0;
    for (int j = 0; j < NT; ++j) {
      mbar_wait(&kv_full[st], ph);
      float s[FT_BN / 2];
      {
        const uint64_t dk = wgmma_desc_k_sw128(smem_u32(sK + st * FT_TILE));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < FT_D / 16; ++k) wgmma_bf16<FT_BN>(s, dq + 2 * k, dk + 2 * k, k != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
      }
      if (j == 0) {
        // the only second pass: the row maximum of the first tile anchors the reference exponent
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float mx = -1e30f;
#pragma unroll
          for (int c = 0; c < FT_BN / 8; ++c) mx = fmaxf(mx, fmaxf(s[4 * c + 2 * e], s[4 * c + 2 * e + 1]));
          mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
          mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
          mb[e] = mx * sl2;
        }
      }
      float scale_due[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        scale_due[e] = __int_as_float((127 - pending[e]) << 23);     // 2^-pending (1.0 when nothing is due)
        mb[e] += (float)pending[e];
      }
      // one pass: p = 2^(s * sl2 - mb) -> packed bf16 (the A fragments of P V), running maximum of the packed values
      uint32_t pa[FT_BN / 16][4];
      float pm[2] = {0.f, 0.f};
      float ts[2] = {0.f, 0.f};
#pragma unroll
      for (int c = 0; c < FT_BN / 8; ++c) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float p0 = ex2_approx(fmaf(s[4 * c + 2 * e], sl2, -mb[e]));
          const float p1 = ex2_approx(fmaf(s[4 * c + 2 * e + 1], sl2, -mb[e]));
          const uint32_t pp = pack_bf16x2(p0, p1);
          const float2 pr = unpack_bf16x2(pp);
          pm[e] = fmaxf(pm[e], fmaxf(pr.x, pr.y));
          ts[e] += pr.x + pr.y;
          pa[c >> 1][(c & 1) * 2 + e] = pp;
        }
      }
      // exact power-of-two rescale of this row's O and L (rows with nothing due multiply by 1)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        lsum[e] = fmaf(lsum[e], scale_due[e], ts[e]);
#pragma unroll
        for (int c = 0; c < FT_D / 8; ++c) {
          o[4 * c + 2 * e] *= scale_due[e];
          o[4 * c + 2 * e + 1] *= scale_due[e];
        }
      }
      {
        const uint32_t v0 = smem_u32(sV + st * FT_TILE);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < FT_BN / 16; ++k)           // 16 keys per step: +16 key rows = 2048 B in the V tile (MN-major)
          wgmma_m64n64k16_rs_tb(o, pa[k], wgmma_desc_mn_sw128(v0 + k * 16 * 128), 1u);
        wgmma_commit();
        wgmma_wait<0>();
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&kv_empty[st]);       // every MMA reading K_j / V_j has completed
      if (++st == FT_NST) { st = 0; ph ^= 1; }
      // did this tile outgrow the reference?  (p <= 2^8 keeps bf16 / fp32 comfortably in range)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float m = fmaxf(pm[e], __shfl_xor_sync(0xffffffffu, pm[e], 1));
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
        pending[e] = m > FT_TAU ? (int)((__float_as_uint(m) >> 23) & 0xff) - 127 : 0;
      }
    }
    // O / L
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      float l = lsum[e];
      l += __shfl_xor_sync(0xffffffffu, l, 1);
      l += __shfl_xor_sync(0xffffffffu, l, 2);
      const float inv = 1.f / l;
      const int r = wg * 64 + 16 * w + (lane >> 2) + 8 * e;
      __nv_bfloat16* orow = out + (size_t)(q0 + r) * ldo + h * FT_D + 2 * t4;
#pragma unroll
      for (int c = 0; c < FT_D / 8; ++c)
        *reinterpret_cast<uint32_t*>(orow + 8 * c) = pack_bf16x2(o[4 * c + 2 * e] * inv, o[4 * c + 2 * e + 1] * inv);
    }
  }
}

static int encode_rows_map(CUtensorMap* map, const void* base, int ld, long long rows, int cols) {
  return tmap_rows_bf16(map, base, ld, rows, cols, FT_BN);
}

// Returns PGT_ERR_UNSUPPORTED when the shape is not covered (caller falls back to the mma.sync kernel).
int mha_tc_launch(const void* q, int ldq, const void* k, int ldk, const void* v, int ldv, int clips, int L, int heads,
                  int d, void* out, int ldo, cudaStream_t stream) {
  if (d != FT_D || L % FT_BM != 0) return PGT_ERR_UNSUPPORTED;
  auto al = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  if (!al(q) || !al(k) || !al(v) || !al(out) || ldq % 8 || ldk % 8 || ldv % 8 || ldo % 8) return PGT_ERR_UNSUPPORTED;
  CUtensorMap tq, tk, tv;
  const long long rows = (long long)clips * L;
  int rc = encode_rows_map(&tq, q, ldq, rows, heads * d);
  if (rc == PGT_OK) rc = encode_rows_map(&tk, k, ldk, rows, heads * d);
  if (rc == PGT_OK) rc = encode_rows_map(&tv, v, ldv, rows, heads * d);
  if (rc != PGT_OK) return rc;
  static PerDeviceOnce once;
  PGT_CUDA_OK(once.run([] { return cudaFuncSetAttribute(mha_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FT_SMEM); }));
  dim3 grid(L / FT_BM, heads, clips);
  mha_tc_kernel<<<grid, FT_THREADS, FT_SMEM, stream>>>(tq, tk, tv, L, reinterpret_cast<__nv_bfloat16*>(out), ldo);
  PGT_LAUNCH_OK();
  return PGT_OK;
}

}  // namespace pgt
