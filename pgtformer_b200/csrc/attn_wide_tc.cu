// Global attention forward for wide heads (d = 256 / 512, no mask) on wgmma, sm_90a: the core of TDRQVAE's dense
// AttnBlock (softmax(q k^T d^-1/2) v over all H*W tokens of a frame, one head of width C = d).
//
// One CTA = one (clip, head) and one query tile; three warpgroups:
//   warpgroup 2     TMA producer (one elected lane; the warpgroup gives its registers back with setmaxnreg): the Q tile
//                   once, then K_j / V_j tiles through a 2-deep ring.  Every tile is stored as [rows x 64] bf16 column
//                   chunks, 128-byte swizzled, one TMA box each.
//   warpgroups 0,1  consumers (raised to 240 registers): each owns a 64-row x 256-column slice of O as fp32 wgmma
//                   accumulators (128 registers per thread).
//     d = 256: the two warpgroups take query rows [0, 64) and [64, 128) of a 128-query tile; 64-key K/V tiles.
//     d = 512: both take the same 64 queries, warpgroup w the O columns [256 w, 256 w + 256).  Each computes the partial
//              S = Q K_j^T over its own 256 channels; the partials are exchanged through shared memory and added
//              (s_own + s_other: fp32 addition commutes, so both warpgroups hold the same S and run the same softmax).
//              32-key K/V tiles.
//   Softmax as in mha_tc.cu: p = 2^(s d^-1/2 log2(e) - m_ref) with a per-row reference exponent m_ref, an integer set
//   from the first tile's row maximum and only raised by whole powers of two (the rescale of O and L is exact).  Here
//   the raise is decided from each tile's row maximum BEFORE exponentiating (when it exceeds m_ref by more than 8), so
//   no score range can overflow p; for these widths the extra pass over S is small next to the two MMAs.  P is packed
//   to bf16 in registers as the A operand of O += P V_j (wgmma 64 x 256 x 16, V read MN-major from its chunks), and L
//   sums exactly the bf16 P that the numerator uses.
//   Frames are consecutive row blocks of one buffer: keys at index >= L of a partial last tile belong to the next frame
//   (or are TMA zero fill) and are masked to -inf by index; query rows >= L are computed and not stored.  Any L >= 1.
#include <cudaTypedefs.h>

#include "common.cuh"
#include "tmap.cuh"
#include "ptx.cuh"

namespace pgt {

template <int D>
struct WideCfg {
  static constexpr int BM = D == 256 ? 128 : 64;                 // queries per CTA
  static constexpr int BN = D == 256 ? 64 : 32;                  // keys per K/V tile
  static constexpr int NST = 2;                                  // K/V ring depth
  static constexpr int Q_BYTES = BM * D * 2;
  static constexpr int KV_BYTES = BN * D * 2;                    // one K (or V) tile
  static constexpr int X_BYTES = D == 512 ? 2 * 2 * 64 * BN * 4 : 0;   // S exchange [tile parity][warpgroup][64 x BN] fp32
  static constexpr int SMEM = Q_BYTES + NST * 2 * KV_BYTES + X_BYTES + 256 + 1024;
  static constexpr float SL2 = (D == 256 ? 0.0625f : 0.044194173824159216f) * 1.4426950408889634f;   // d^-1/2 log2(e)
};
constexpr int WA_THREADS = 384;
constexpr float WA_RAISE = 8.f;             // a tile row maximum more than 2^8 above the reference raises the reference

template <int D>
__global__ void __launch_bounds__(WA_THREADS, 1)
attn_wide_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                 const __grid_constant__ CUtensorMap tmV, int L, __nv_bfloat16* __restrict__ out, int ldo) {
  using C = WideCfg<D>;
  constexpr int BM = C::BM, BN = C::BN, NST = C::NST;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;                                            // [D/64 chunks][BM x 128 B]
  uint8_t* sK = sQ + C::Q_BYTES;                                 // [NST][D/64 chunks][BN x 128 B]
  uint8_t* sV = sK + NST * C::KV_BYTES;                          // [NST][D/64 chunks][BN x 128 B]
  float4* sX = reinterpret_cast<float4*>(sV + NST * C::KV_BYTES);
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + NST * C::KV_BYTES + C::X_BYTES);
  uint64_t* q_full = bars;                                       // [1]
  uint64_t* kv_full = bars + 1;                                  // [NST]
  uint64_t* kv_empty = kv_full + NST;                            // [NST] one arrive per consumer warp

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = blockIdx.y;
  const int qt = blockIdx.x * BM;                                // first query of this CTA inside its frame
  const int kv0 = blockIdx.z * L;                                // first row of this frame
  const int NT = (L + BN - 1) / BN;

  if (threadIdx.x == 256) {
    tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV);
    mbar_init(q_full, 1);
    for (int i = 0; i < NST; ++i) { mbar_init(&kv_full[i], 1); mbar_init(&kv_empty[i], 8); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= 8) {
    // ------------------------------------------------------------------ TMA producer
    setmaxnreg_dec<24>();
    if (warp == 8) {
      if (elect_one()) {
        mbar_arrive_expect_tx(q_full, C::Q_BYTES);
#pragma unroll
        for (int c = 0; c < D / 64; ++c) tma_load_2d(sQ + c * BM * 128, &tmQ, q_full, h * D + 64 * c, kv0 + qt);
      }
      __syncwarp();
      int st = 0;
      uint32_t ph = 0;
      // NST more waits than loads: the drain waits (bounded) until the consumers have released every tile, so a
      // transaction that never completes (an expect_tx byte count that disagrees with the boxes) traps the launch
      // instead of leaving the consumers' unbounded waits spinning
      for (int j = 0; j < NT + NST; ++j) {
        mbar_wait(&kv_empty[st], ph ^ 1);
        if (j < NT && elect_one()) {
          mbar_arrive_expect_tx(&kv_full[st], 2 * C::KV_BYTES);
#pragma unroll
          for (int c = 0; c < D / 64; ++c) {
            tma_load_2d(sK + st * C::KV_BYTES + c * BN * 128, &tmK, &kv_full[st], h * D + 64 * c, kv0 + j * BN);
            tma_load_2d(sV + st * C::KV_BYTES + c * BN * 128, &tmV, &kv_full[st], h * D + 64 * c, kv0 + j * BN);
          }
        }
        __syncwarp();
        if (++st == NST) { st = 0; ph ^= 1; }
      }
    }
  } else {
    // ------------------------------------------------------------------ attention warpgroups
    setmaxnreg_inc<240>();
    const int wg = warp >> 2, w = warp & 3;
    const int t4 = lane & 3;
    const int qrow = D == 256 ? 64 * wg : 0;                     // this warpgroup's first query row in the tile
    const int cbase = D == 512 ? 4 * wg : 0;                     // first 64-column chunk of its 256 channels
    const uint32_t q_addr = smem_u32(sQ) + cbase * BM * 128 + qrow * 128;
    float o[128];                                                // O: rows (g, g + 8) of the warp's 16, 256 columns
    float mb[2] = {0.f, 0.f};                                    // reference exponent per row (integer, log2 domain)
    float lsum[2] = {0.f, 0.f};                                  // this lane's share of the row sums of the bf16 P
#pragma unroll
    for (int i = 0; i < 128; ++i) o[i] = 0.f;
    // unbounded waits here (see mbar_wait_spin): a transaction that never completes leaves the producer's bounded drain
    // waiting for this stage's release, and its trap ends the launch
    mbar_wait_spin(q_full, 0);
    int st = 0;
    uint32_t ph = 0;
    for (int j = 0; j < NT; ++j) {
      mbar_wait_spin(&kv_full[st], ph);
      float s[BN / 2];
      {
        const uint32_t k_addr = smem_u32(sK + st * C::KV_BYTES) + cbase * BN * 128;
        wgmma_fence();
#pragma unroll
        for (int c = 0; c < 4; ++c)
#pragma unroll
          for (int kk = 0; kk < 4; ++kk)                         // 16 channels per step: +32 B inside a 128 B row
            wgmma_bf16<BN>(s, wgmma_desc_k_sw128(q_addr + c * BM * 128 + 32 * kk),
                           wgmma_desc_k_sw128(k_addr + c * BN * 128 + 32 * kk), (c | kk) != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
      }
      if constexpr (D == 512) {
        // thread t of either warpgroup holds the same S elements: exchange the partials fragment-wise
        const int tid = threadIdx.x & 127;
        float4* mine = sX + ((j & 1) * 2 + wg) * (BN / 8) * 128;
        const float4* other = sX + ((j & 1) * 2 + (wg ^ 1)) * (BN / 8) * 128;
#pragma unroll
        for (int i = 0; i < BN / 8; ++i) mine[i * 128 + tid] = make_float4(s[4 * i], s[4 * i + 1], s[4 * i + 2], s[4 * i + 3]);
        named_bar_sync(1, 256);          // also orders this tile's reads of the other parity before its next overwrite
#pragma unroll
        for (int i = 0; i < BN / 8; ++i) {
          const float4 f = other[i * 128 + tid];
          s[4 * i] += f.x; s[4 * i + 1] += f.y; s[4 * i + 2] += f.z; s[4 * i + 3] += f.w;
        }
      }
      if ((j + 1) * BN > L) {
        // partial last tile: keys past the frame are -inf (exp -> 0), never TMA's zero fill or the next frame's rows
        const int kb = j * BN + 2 * t4;
#pragma unroll
        for (int c = 0; c < BN / 8; ++c)
#pragma unroll
          for (int e = 0; e < 2; ++e)
#pragma unroll
            for (int b = 0; b < 2; ++b)
              if (kb + 8 * c + b >= L) s[4 * c + 2 * e + b] = -INFINITY;
      }
      float scale_due[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float mx = -INFINITY;
#pragma unroll
        for (int c = 0; c < BN / 8; ++c) mx = fmaxf(mx, fmaxf(s[4 * c + 2 * e], s[4 * c + 2 * e + 1]));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        const float mt = mx * C::SL2;
        if (j == 0) {
          mb[e] = ceilf(mt);
          scale_due[e] = 1.f;
        } else {
          const float n = mt - mb[e] > WA_RAISE ? ceilf(mt - mb[e]) : 0.f;
          mb[e] += n;
          scale_due[e] = n >= 127.f ? 0.f : __int_as_float((127 - (int)n) << 23);    // 2^-n
        }
      }
      // p = 2^(s * sl2 - mb) -> packed bf16 (the A fragments of P V); row sums over exactly those bf16 values
      uint32_t pa[BN / 16][4];
      float ts[2] = {0.f, 0.f};
#pragma unroll
      for (int c = 0; c < BN / 8; ++c) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float p0 = ex2_approx(fmaf(s[4 * c + 2 * e], C::SL2, -mb[e]));
          const float p1 = ex2_approx(fmaf(s[4 * c + 2 * e + 1], C::SL2, -mb[e]));
          const uint32_t pp = pack_bf16x2(p0, p1);
          const float2 pr = unpack_bf16x2(pp);
          ts[e] += pr.x + pr.y;
          pa[c >> 1][(c & 1) * 2 + e] = pp;
        }
      }
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        lsum[e] = fmaf(lsum[e], scale_due[e], ts[e]);
#pragma unroll
        for (int c = 0; c < 32; ++c) {
          o[4 * c + 2 * e] *= scale_due[e];
          o[4 * c + 2 * e + 1] *= scale_due[e];
        }
      }
      {
        const uint32_t v_addr = smem_u32(sV + st * C::KV_BYTES) + cbase * BN * 128;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BN / 16; ++k)              // 16 keys per step: +16 rows = 2048 B in every V chunk
          wgmma_m64n256k16_rs_tb(o, pa[k], wgmma_desc_mn_sw128(v_addr + k * 2048, BN * 128), 1u);
        wgmma_commit();
        wgmma_wait<0>();
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&kv_empty[st]);       // every MMA reading K_j / V_j has completed
      if (++st == NST) { st = 0; ph ^= 1; }
    }
    // O / L, rows inside the frame only
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      float l = lsum[e];
      l += __shfl_xor_sync(0xffffffffu, l, 1);
      l += __shfl_xor_sync(0xffffffffu, l, 2);
      const float inv = 1.f / l;
      const int r = qt + qrow + 16 * w + (lane >> 2) + 8 * e;
      if (r < L) {
        __nv_bfloat16* orow = out + (size_t)(kv0 + r) * ldo + h * D + 64 * cbase + 2 * t4;
#pragma unroll
        for (int c = 0; c < 32; ++c)
          *reinterpret_cast<uint32_t*>(orow + 8 * c) = pack_bf16x2(o[4 * c + 2 * e] * inv, o[4 * c + 2 * e + 1] * inv);
      }
    }
  }
}

template <int D>
static int attn_wide_run(const void* q, int ldq, const void* k, int ldk, const void* v, int ldv, int clips, int L,
                         int heads, void* out, int ldo, cudaStream_t stream) {
  using C = WideCfg<D>;
  CUtensorMap tq, tk, tv;
  const long long rows = (long long)clips * L;
  int rc = tmap_rows_bf16(&tq, q, ldq, rows, heads * D, C::BM);
  if (rc == PGT_OK) rc = tmap_rows_bf16(&tk, k, ldk, rows, heads * D, C::BN);
  if (rc == PGT_OK) rc = tmap_rows_bf16(&tv, v, ldv, rows, heads * D, C::BN);
  if (rc != PGT_OK) return rc;
  static PerDeviceOnce once;
  PGT_CUDA_OK(once.run([] {
    return cudaFuncSetAttribute(attn_wide_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM);
  }));
  dim3 grid(ceil_div(L, C::BM), heads, clips);
  attn_wide_kernel<D><<<grid, WA_THREADS, C::SMEM, stream>>>(tq, tk, tv, L, reinterpret_cast<__nv_bfloat16*>(out), ldo);
  PGT_LAUNCH_OK();
  return PGT_OK;
}

// d = 256 / 512 (any L >= 1); PGT_ERR_UNSUPPORTED for other widths and for operands TMA cannot address.
int attn_wide_launch(const void* q, int ldq, const void* k, int ldk, const void* v, int ldv, int clips, int L, int heads,
                     int d, void* out, int ldo, cudaStream_t stream) {
  auto al = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  if (!al(q) || !al(k) || !al(v) || !al(out) || ldq % 8 || ldk % 8 || ldv % 8 || ldo % 8) return PGT_ERR_UNSUPPORTED;
  if (d == 256) return attn_wide_run<256>(q, ldq, k, ldk, v, ldv, clips, L, heads, out, ldo, stream);
  if (d == 512) return attn_wide_run<512>(q, ldq, k, ldk, v, ldv, clips, L, heads, out, ldo, stream);
  return PGT_ERR_UNSUPPORTED;
}

}  // namespace pgt
