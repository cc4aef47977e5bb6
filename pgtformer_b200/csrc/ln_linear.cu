// LayerNorm fused into the GEMM that consumes it (C = 256):   out[T, N] = LN(x)[T, 256] * W[N, 256]^T + b
// Replaces norm1 + the q / kv projections of WindowAttention3D (modules/rstt_layers.py:116-132,176-188, fused into one
// [3C, C] weight at load): the normalised token matrix is never written to HBM — x is read once, LN happens in shared
// memory in place, and the same tile is the A operand of all N / 256 column blocks.
//
// Per CTA, persistent over 128-token tiles (448 threads):
//   warps 0..7  two consumer warpgroups: warpgroup h multiplies rows [64h, 64h + 64) of the tile with one 128-column
//               weight block at a time (wgmma 64 x 128 x 16, fp32 accumulators in registers), then adds the bias and
//               writes bf16 pairs straight from the accumulator fragments into the swizzled 64-column staging panels
//   warp 8      TMA producer of the weight k-blocks ([128 x 64] each, 4-deep ring; N/128 x 4 per tile)
//   warp 9      DMA: TMA load of x tiles into the buffer the MMAs of two tiles ago have released, TMA store of each
//               finished [128 x 64] panel
//   warps 10..13 LayerNorm of the NEXT x tile in place, one thread per row (no cross-thread exchange), concurrent with
//               the epilogues and MMAs of the current tile
//
// Two x buffers (round 2, second pass).  A device timeline of the single-buffer version (clock64 stamps, T = 786432):
// per 22.4 k-cycle tile the tensor pipe was busy 8.1 k — the x load could only be issued once the tile's last MMA had
// retired and then took 8.5 k cycles (it queues behind the output stores every CTA has just issued), LayerNorm another
// 4.4 k, all of it serial.  Now x(i+1) is loaded and normalised (by warps of its own: with the LayerNorm on the epilogue
// warps the tile was still bounded by LayerNorm + three epilogues, 16.7 k) while tile i is multiplied; the shared memory
// comes from the staging buffer (two 64-column panels instead of two 128-column halves) and the weight ring (2 x 32 KB).
#include <cudaTypedefs.h>

#include <cstdio>

#include "common.cuh"
#include "tmap.cuh"
#include "ptx.cuh"

namespace pgt {

constexpr int LL_C = 256;
constexpr int LL_BM = 128;
constexpr int LL_SUB = LL_BM * 128;            // one [128 x 64] bf16 sub-tile: 16 KB
constexpr int LL_BN = 128;                     // weight block (columns) per wgmma pass
constexpr int LL_WST = 4;                      // weight ring depth
constexpr int LL_WBYTES = LL_BN * 128;         // one [128 x 64] weight k-block: 16 KB
constexpr int LL_THREADS = 448;
constexpr int LL_SMEM = 8 * LL_SUB /*two x / A tiles*/ + 2 * LL_SUB /*staging panels*/ + LL_WST * LL_WBYTES + 256;
static_assert(LL_SMEM <= 232448, "ln_linear smem budget");

struct LnLinearParams {
  int T, m_tiles, nb;   // nb = N / 256 column blocks
  const float* ln_g;
  const float* ln_b;
  float eps;
  const float* bias;    // [N]
};

__global__ void __launch_bounds__(LL_THREADS, 1)
ln_linear_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmO,
                 const __grid_constant__ CUtensorMap tmW, const LnLinearParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];     // no static smem in this kernel: the window starts 1024-aligned
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  uint8_t* sX = smem;                           // [2] x tile -> LN(x): the A operand of every column block
  uint8_t* sO = sX + 8 * LL_SUB;                // [2] finished [128 x 64] panels (ping-pong)
  uint8_t* sW = sO + 2 * LL_SUB;                // weight ring
  uint64_t* bars = reinterpret_cast<uint64_t*>(sW + LL_WST * LL_WBYTES);
  uint64_t* x_full = bars;           // [2] DMA -> LayerNorm warps
  uint64_t* sx_free = bars + 2;      // [2] consumers (one arrive per warp, after the tile's last MMAs) -> DMA
  uint64_t* y_ready = bars + 4;      // [2] LayerNorm warps (128) -> consumers
  uint64_t* so_free = bars + 6;      // [2] DMA (store has read staging panel s) -> consumers
  uint64_t* out_ready = bars + 8;    // [2] consumers (256) -> DMA
  uint64_t* w_full = bars + 10;      // [LL_WST]
  uint64_t* w_empty = w_full + LL_WST;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmX); tma_prefetch_desc(&tmO); tma_prefetch_desc(&tmW);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&x_full[i], 1); mbar_init(&sx_free[i], 8); mbar_init(&y_ready[i], 128);
      mbar_init(&so_free[i], 1); mbar_init(&out_ready[i], 256);
    }
    for (int i = 0; i < LL_WST; ++i) { mbar_init(&w_full[i], 1); mbar_init(&w_empty[i], 8); }
    fence_barrier_init();
  }
  __syncthreads();
  const int NB = p.nb;
  const int NB2 = NB * (LL_C / LL_BN);

  if (warp == 8) {
    // ------------------------------------------------------------------ weight producer
    int st = 0;
    uint32_t ph = 0;
    for (int tile = blockIdx.x; tile < p.m_tiles; tile += gridDim.x) {
      for (int j = 0; j < NB2; ++j) {
        for (int kb = 0; kb < 4; ++kb) {
          mbar_wait(&w_empty[st], ph ^ 1);
          if (elect_one()) {
            mbar_arrive_expect_tx(&w_full[st], LL_WBYTES);
            tma_load_2d(sW + st * LL_WBYTES, &tmW, &w_full[st], kb * 64, j * LL_BN);
          }
          __syncwarp();
          if (++st == LL_WST) { st = 0; ph ^= 1; }
        }
      }
    }
  } else if (warp < 8) {
    // ------------------------------------------------------------------ consumer warpgroups
    const int wg = warp >> 2, w = warp & 3;
    const int t4 = lane & 3;
    const uint32_t so = smem_u32(sO);
    int st = 0;
    uint32_t ph = 0;
    int it = 0;
    int n = 0;                                           // running panel number: staging buffer n & 1, its (n >> 1)-th use
    for (int tile = blockIdx.x; tile < p.m_tiles; tile += gridDim.x, ++it) {
      const int xb = it & 1;
      mbar_wait(&y_ready[xb], (it >> 1) & 1);
      const uint32_t a_rows = smem_u32(sX + xb * 4 * LL_SUB) + wg * 64 * 128;
      for (int j = 0; j < NB2; ++j) {
        float acc[LL_BN / 2];
        int prev = -1;
        for (int kb = 0; kb < 4; ++kb) {
          mbar_wait(&w_full[st], ph);
          const uint64_t da = wgmma_desc_k_sw128(a_rows + kb * LL_SUB);
          const uint64_t db = wgmma_desc_k_sw128(smem_u32(sW) + st * LL_WBYTES);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < 4; ++k) wgmma_bf16<LL_BN>(acc, da + 2 * k, db + 2 * k, (kb | k) != 0 ? 1u : 0u);
          wgmma_commit();
          wgmma_wait<1>();
          if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&w_empty[prev]); }
          prev = st;
          if (++st == LL_WST) { st = 0; ph ^= 1; }
        }
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) {
          mbar_arrive(&w_empty[prev]);
          if (j == NB2 - 1) mbar_arrive(&sx_free[xb]);   // every MMA that reads this x buffer has retired
        }
        // ---- acc + bias -> bf16 -> two 64-column staging panels: fragment column pair (2 t4, 2 t4 + 1) of 8-column
        // chunk jj is one 4-byte word of the swizzled row
#pragma unroll
        for (int pp = 0; pp < LL_BN / 64; ++pp, ++n) {
          const int sb = n & 1;
          const float* bias = p.bias + j * LL_BN + pp * 64 + 2 * t4;
          float2 bv[8];                                // requested before the wait
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) bv[jj] = __ldg(reinterpret_cast<const float2*>(bias + 8 * jj));
          mbar_wait(&so_free[sb], ((n >> 1) & 1) ^ 1);   // the store that last used this panel has read it
#pragma unroll
          for (int hr = 0; hr < 2; ++hr) {
            const int r = wg * 64 + w * 16 + (lane >> 2) + 8 * hr;
            const uint32_t dst = so + sb * LL_SUB + r * 128 + t4 * 4;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
              const int f = 4 * (pp * 8 + jj) + 2 * hr;
              const uint32_t o = pack_bf16x2(acc[f] + bv[jj].x, acc[f + 1] + bv[jj].y);
              asm volatile("st.shared.b32 [%0], %1;" ::"r"(dst + ((jj ^ (r & 7)) << 4)), "r"(o) : "memory");
            }
          }
          fence_proxy_async();
          mbar_arrive(&out_ready[sb]);
        }
      }
    }
  } else if (warp == 9) {
    // ------------------------------------------------------------------ DMA warp
    int it = 0;
    int pending = -1;                                  // staging panel of the newest committed store (not yet released)
    if (lane == 0) {
      for (int t = 0; t < 2; ++t) {
        const int tile = blockIdx.x + t * gridDim.x;
        if (tile < p.m_tiles) {
          mbar_arrive_expect_tx(&x_full[t], 4 * LL_SUB);
          for (int kb = 0; kb < 4; ++kb) tma_load_2d(sX + (t * 4 + kb) * LL_SUB, &tmX, &x_full[t], kb * 64, tile * LL_BM);
        }
      }
    }
    __syncwarp();
    for (int tile = blockIdx.x; tile < p.m_tiles; tile += gridDim.x, ++it) {
      const int xb = it & 1;
      for (int j = 0; j < NB; ++j) {
        const int g = it * NB + j;
        for (int pp = 0; pp < 4; ++pp) {
          if (j == NB - 1 && pp == 4 - LL_BN / 64) {
            // this tile's x buffer is free once the MMAs of its last 128-column block have retired: fetch the tile after
            // next.  The consumers release it before they write that block's panels, and only after the panels before
            // them have been stored (their staging slots are needed), so the wait sits exactly here.
            const int nt = tile + 2 * gridDim.x;
            if (nt < p.m_tiles) {
              mbar_wait(&sx_free[xb], (it >> 1) & 1);
              if (lane == 0) {
                mbar_arrive_expect_tx(&x_full[xb], 4 * LL_SUB);
                for (int kb = 0; kb < 4; ++kb) tma_load_2d(sX + (xb * 4 + kb) * LL_SUB, &tmX, &x_full[xb], kb * 64, nt * LL_BM);
              }
              __syncwarp();
            }
          }
          const int n = g * 4 + pp;
          const int sb = n & 1;
          mbar_wait(&out_ready[sb], (n >> 1) & 1);
          if (lane == 0) {
            tma_store_2d(&tmO, sO + sb * LL_SUB, j * LL_C + pp * 64, tile * LL_BM);
            bulk_commit();
            if (pending >= 0) {
              bulk_wait_read<1>();                       // the store before this one has read its panel
              mbar_arrive(&so_free[pending]);
            }
          }
          pending = sb;
          __syncwarp();
        }
      }
    }
    if (lane == 0) bulk_wait0();
  } else {
    // ------------------------------------------------------------------ LayerNorm warps (10..13): thread = row
    const int r = (warp - 10) * 32 + lane;
    const bool affine = p.ln_g != nullptr;             // nullptr: gamma / beta folded into W / bias by the caller
    int t = 0;
    for (int tile = blockIdx.x; tile < p.m_tiles; tile += gridDim.x, ++t) {
      const uint32_t xb = smem_u32(sX) + (t & 1) * 4 * LL_SUB + r * 128;
      mbar_wait(&x_full[t & 1], (t >> 1) & 1);
      float s = 0.f, q = 0.f;
#pragma unroll
      for (int sub = 0; sub < 4; ++sub) {
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          uint4 u;
          asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(u.x), "=r"(u.y), "=r"(u.z), "=r"(u.w)
                       : "r"(xb + sub * LL_SUB + ((c ^ (r & 7)) << 4)) : "memory");
          const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), cc = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
          s += (a.x + a.y) + (b.x + b.y) + (cc.x + cc.y) + (d.x + d.y);
          q += a.x * a.x + a.y * a.y + b.x * b.x + b.y * b.y + cc.x * cc.x + cc.y * cc.y + d.x * d.x + d.y * d.y;
        }
      }
      const float mean = s * (1.f / LL_C);
      const float var = fmaxf(q * (1.f / LL_C) - mean * mean, 0.f);
      const float rstd = rsqrtf(var + p.eps);
      const float nm = -mean * rstd;
#pragma unroll 1
      for (int sub = 0; sub < 4; ++sub) {
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          const uint32_t addr = xb + sub * LL_SUB + ((c ^ (r & 7)) << 4);
          uint4 u;
          asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(u.x), "=r"(u.y), "=r"(u.z), "=r"(u.w) : "r"(addr) : "memory");
          const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), cc = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
          const float v[8] = {a.x, a.y, b.x, b.y, cc.x, cc.y, d.x, d.y};
          float y[8];
          if (affine) {
            const int col = sub * 64 + c * 8;
            const float4 g0 = __ldg(reinterpret_cast<const float4*>(p.ln_g + col)), g1 = __ldg(reinterpret_cast<const float4*>(p.ln_g + col + 4));
            const float4 e0 = __ldg(reinterpret_cast<const float4*>(p.ln_b + col)), e1 = __ldg(reinterpret_cast<const float4*>(p.ln_b + col + 4));
            const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
            const float ee[8] = {e0.x, e0.y, e0.z, e0.w, e1.x, e1.y, e1.z, e1.w};
#pragma unroll
            for (int j = 0; j < 8; ++j) y[j] = fmaf(fmaf(v[j], rstd, nm), gg[j], ee[j]);
          } else {
#pragma unroll
            for (int j = 0; j < 8; ++j) y[j] = fmaf(v[j], rstd, nm);
          }
          const uint32_t ox = pack_bf16x2(y[0], y[1]), oy = pack_bf16x2(y[2], y[3]), oz = pack_bf16x2(y[4], y[5]), ow = pack_bf16x2(y[6], y[7]);
          asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(ox), "r"(oy), "r"(oz), "r"(ow) : "memory");
        }
      }
      fence_proxy_async();
      mbar_arrive(&y_ready[t & 1]);
    }
  }
}

static int ll_enc2d(CUtensorMap* map, const void* base, int ld, long long rows, int cols, int box_rows) {
  return tmap_rows_bf16(map, base, ld, rows, cols, box_rows);
}

}  // namespace pgt

using namespace pgt;

extern "C" int pgt_ln_linear_bf16(const void* x, int ldx, int T, int C, const float* ln_g, const float* ln_b, float eps,
                                  const void* W, int ldw, int N, const float* bias, void* out, int ldo, void* stream) {
  PGT_CHECK_ARG(x && out && W && bias && T > 0 && N > 0 && ((ln_g == nullptr) == (ln_b == nullptr)));   // both null: no affine
  if (C != LL_C || (N % LL_C) != 0) return PGT_ERR_UNSUPPORTED;
  auto al = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  PGT_CHECK_ARG(al(x) && al(out) && al(W) && ldx % 8 == 0 && ldo % 8 == 0 && ldw % 8 == 0 && ldw >= C && ldo >= N);
  CUtensorMap tx, to, tw;
  int rc = ll_enc2d(&tx, x, ldx, T, C, LL_BM);
  if (rc == PGT_OK) rc = ll_enc2d(&to, out, ldo, T, N, LL_BM);
  if (rc == PGT_OK) rc = ll_enc2d(&tw, W, ldw, N, C, LL_BN);
  if (rc != PGT_OK) return rc;
  static PerDeviceOnce once;
  PGT_CUDA_OK(once.run([] { return cudaFuncSetAttribute(ln_linear_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, LL_SMEM); }));
  LnLinearParams p{};
  p.T = T; p.m_tiles = ceil_div(T, LL_BM); p.nb = N / LL_C;
  p.ln_g = ln_g; p.ln_b = ln_b; p.eps = eps; p.bias = bias;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int grid = p.m_tiles < num_sms() ? p.m_tiles : num_sms();
  {
    char desc[64];
    if (prof_enabled()) snprintf(desc, sizeof(desc), "ln_linear M%d N%d K256", T, N);
    ProfScope ps(PGT_PROF_GEMM, 2.0 * (double)T * N * C, st, desc);
    ln_linear_kernel<<<grid, LL_THREADS, LL_SMEM, st>>>(tx, to, tw, p);
  }
  PGT_LAUNCH_OK();
  return PGT_OK;
}
