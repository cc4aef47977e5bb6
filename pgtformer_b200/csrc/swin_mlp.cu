// Fused Swin MLP half-block on wgmma (C = 256):   out = x + W2 * GELU(W1 * LN(x) + b1) + b2
// Replaces LayerNorm(norm2) + Mlp(fc1, exact GELU, fc2) + residual of VSTSREncoderTransformerBlock
// (modules/rstt_layers.py:116-132,335-336): five HBM passes over the token matrix (LN r/w, fc1 r/w, fc2 r+r/w)
// become two (read x, write out); the 128 x 256 hidden tile never leaves the SM.
//
// Per CTA, persistent over 128-token tiles (320 threads):
//   warps 0..7    two consumer warpgroups; warpgroup h owns rows [64h, 64h + 64) of the tile through the whole chain
//                 LN -> GEMM1 -> GELU -> GEMM2 -> +b2 +x, so the in-place rewrites of the tile buffer only ever wait for
//                 the warpgroup's own MMAs: LayerNorm of its rows in place (two threads per row), wgmma 64 x 256 x 16
//                 (fp32 accumulators in registers), GELU epilogue written back in place as the A operand of GEMM2, final
//                 epilogue acc + b2 + x in place.  Accumulators reach the row-per-thread epilogues through a 64 x 64
//                 fp32 exchange per warpgroup.  One 64 KB buffer carries x -> LN(x) -> hidden -> x (again) -> out.
//   warp 8        TMA producer of the weight k-blocks (W1 / W2, 256 x 64 each, 3-deep ring)
//   warp 9        DMA: TMA load of the x tile, re-fetch of x (an L2 hit) for the residual once GEMM2 has consumed the
//                 buffer, TMA store of the finished tile
#include <cudaTypedefs.h>

#include "common.cuh"
#include "tmap.cuh"
#include "ptx.cuh"
#include "epi_common.cuh"

namespace pgt {

constexpr int SM_C = 256;
constexpr int SM_BM = 128;
constexpr int SM_SUB = SM_BM * 128;            // one [128 x 64] bf16 sub-tile: 16 KB
constexpr int SM_WST = 3;                      // weight ring depth
constexpr int SM_WBYTES = SM_C * 128;          // one [256 x 64] weight k-block: 32 KB
constexpr int SM_THREADS = 320;
constexpr int SM_XLD = 68;                     // accumulator exchange pitch (fp32)
constexpr int SM_XCH = SM_BM * SM_XLD * 4;
constexpr int SM_SMEM = 4 * SM_SUB /*tile*/ + SM_WST * SM_WBYTES + SM_XCH + 128 * 8 /*LN pair exchange*/ + 256;
static_assert(SM_SMEM <= 232448, "swin_mlp smem budget");

struct SwinMlpParams {
  int T, m_tiles;
  const float* ln_g;
  const float* ln_b;
  float eps;
  const float* b1;
  const float* b2;
  float* gn_stats;      // optional [m_tiles][4][32][2]
};

struct SmBars {
  uint64_t x_full, res_full, acc2_done, out_ready;
};

// consumer warpgroups: warp 0..7 of the CTA, warpgroup wg owns rows [64 wg, 64 wg + 64) of every tile
__device__ __forceinline__ void swin_mlp_compute(const SwinMlpParams& p, uint8_t* sX, uint8_t* sW, float* xacc, float2* xln,
                                                 SmBars* bar, uint64_t* w_full, uint64_t* w_empty, int warp, int lane) {
  const int wg = warp >> 2, w = warp & 3;
  const int half = w >> 1;                            // which 32 columns of a 64-column group this thread takes
  const int rl = (w & 1) * 32 + lane;                 // row inside the warpgroup's 64
  const int r = wg * 64 + rl;                         // row of the tile
  const int quad = r >> 5;
  const int bar_id = 1 + wg;                          // named barrier of this warpgroup
  float* xw = xacc + wg * 64 * SM_XLD;                // this warpgroup's exchange rows
  const float* xrow = xw + rl * SM_XLD;
  const uint32_t a_rows = smem_u32(sX) + wg * 64 * 128;
  int st = 0;
  uint32_t ph = 0;
  uint32_t par = 0;
  float acc[SM_C / 2];

  // one GEMM over the four k-blocks of the ring (W1 or W2), A = this warpgroup's rows of the tile buffer
  auto gemm = [&]() {
    int prev = -1;
    for (int kb = 0; kb < 4; ++kb) {
      mbar_wait(&w_full[st], ph);
      const uint64_t da = wgmma_desc_k_sw128(a_rows + kb * SM_SUB);
      const uint64_t db = wgmma_desc_k_sw128(smem_u32(sW) + st * SM_WBYTES);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_bf16<SM_C>(acc, da + 2 * k, db + 2 * k, (kb | k) != 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<1>();
      if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&w_empty[prev]); }
      prev = st;
      if (++st == SM_WST) { st = 0; ph ^= 1; }
    }
    wgmma_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(&w_empty[prev]);
  };
  // columns [64 G, 64 G + 64) of the accumulators -> exchange; then this thread's 32 of them for row r
  auto exchange = [&](auto gc, uint32_t (&v)[32]) {
    constexpr int G = decltype(gc)::value;
    named_bar_sync(bar_id, 128);
    acc_to_smem<64 * G, 64>(acc, xw, SM_XLD, w, lane);
    named_bar_sync(bar_id, 128);
    smem_row_32(xrow + half * 32, v);
  };

  for (int tile = blockIdx.x; tile < p.m_tiles; tile += gridDim.x, par ^= 1) {
    // ---- LayerNorm(x) in place -> A operand of GEMM1 (two threads per row; the halves meet through smem)
    mbar_wait(&bar->x_full, par);
    float s = 0.f, q = 0.f;
#pragma unroll
    for (int sub = 0; sub < 2; ++sub) {
      const uint8_t* src = sX + (half * 2 + sub) * SM_SUB + r * 128;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const uint4 u = *reinterpret_cast<const uint4*>(src + ((c ^ (r & 7)) << 4));
        const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), cc = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
        s += (a.x + a.y) + (b.x + b.y) + (cc.x + cc.y) + (d.x + d.y);
        q += a.x * a.x + a.y * a.y + b.x * b.x + b.y * b.y + cc.x * cc.x + cc.y * cc.y + d.x * d.x + d.y * d.y;
      }
    }
    if (half == 0) xln[r] = make_float2(s, q);
    named_bar_sync(bar_id, 128);
    if (half == 1) {
      const float2 o = xln[r];
      s += o.x; q += o.y;
      xln[r] = make_float2(s, q);
    }
    named_bar_sync(bar_id, 128);
    if (half == 0) {
      const float2 o = xln[r];
      s = o.x; q = o.y;
    }
    const float mean = s * (1.f / SM_C);
    const float var = fmaxf(q * (1.f / SM_C) - mean * mean, 0.f);
    const float rstd = rsqrtf(var + p.eps);
    const float nm = -mean * rstd;
#pragma unroll
    for (int sub = 0; sub < 2; ++sub) {
      const int kb = half * 2 + sub;
      uint8_t* row = sX + kb * SM_SUB + r * 128;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        uint4* ptr = reinterpret_cast<uint4*>(row + ((c ^ (r & 7)) << 4));
        const uint4 u = *ptr;
        const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), cc = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
        const float v[8] = {a.x, a.y, b.x, b.y, cc.x, cc.y, d.x, d.y};
        float y[8];
        if (p.ln_g != nullptr) {
          const int col = kb * 64 + c * 8;
          const float4 g0 = __ldg(reinterpret_cast<const float4*>(p.ln_g + col)), g1 = __ldg(reinterpret_cast<const float4*>(p.ln_g + col + 4));
          const float4 e0 = __ldg(reinterpret_cast<const float4*>(p.ln_b + col)), e1 = __ldg(reinterpret_cast<const float4*>(p.ln_b + col + 4));
          const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
          const float ee[8] = {e0.x, e0.y, e0.z, e0.w, e1.x, e1.y, e1.z, e1.w};
#pragma unroll
          for (int j = 0; j < 8; ++j) y[j] = fmaf(fmaf(v[j], rstd, nm), gg[j], ee[j]);
        } else {                               // gamma / beta folded into W1 / b1 by the caller
#pragma unroll
          for (int j = 0; j < 8; ++j) y[j] = fmaf(v[j], rstd, nm);
        }
        uint4 o;
        o.x = pack_bf16x2(y[0], y[1]); o.y = pack_bf16x2(y[2], y[3]);
        o.z = pack_bf16x2(y[4], y[5]); o.w = pack_bf16x2(y[6], y[7]);
        *ptr = o;
      }
    }
    fence_proxy_async();
    named_bar_sync(bar_id, 128);
    gemm();                                            // GEMM1
    // ---- hidden = GELU(acc + b1) -> A operand of GEMM2 (in place: this warpgroup's GEMM1 has finished reading its rows)
    static_for<0, SM_C / 64>([&](auto gc) {
      constexpr int G = decltype(gc)::value;
      uint32_t v[32];
      exchange(gc, v);
      const int c0 = G * 64 + half * 32;
      const float4* b4 = reinterpret_cast<const float4*>(p.b1 + c0);
      uint8_t* dst = sX + G * SM_SUB + r * 128;
      const int ch0 = half * 4;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float4 ba = __ldg(b4 + 2 * i), bb = __ldg(b4 + 2 * i + 1);
        uint4 o;
        o.x = pack_bf16x2(gelu_erf(__uint_as_float(v[8 * i + 0]) + ba.x), gelu_erf(__uint_as_float(v[8 * i + 1]) + ba.y));
        o.y = pack_bf16x2(gelu_erf(__uint_as_float(v[8 * i + 2]) + ba.z), gelu_erf(__uint_as_float(v[8 * i + 3]) + ba.w));
        o.z = pack_bf16x2(gelu_erf(__uint_as_float(v[8 * i + 4]) + bb.x), gelu_erf(__uint_as_float(v[8 * i + 5]) + bb.y));
        o.w = pack_bf16x2(gelu_erf(__uint_as_float(v[8 * i + 6]) + bb.z), gelu_erf(__uint_as_float(v[8 * i + 7]) + bb.w));
        *reinterpret_cast<uint4*>(dst + (((ch0 + i) ^ (r & 7)) << 4)) = o;
      }
    });
    fence_proxy_async();
    named_bar_sync(bar_id, 128);
    gemm();                                            // GEMM2
    __syncwarp();
    if (lane == 0) mbar_arrive(&bar->acc2_done);
    // ---- out = acc + b2 + x in place over the re-fetched x tile (then TMA-stored by the DMA warp)
    mbar_wait(&bar->res_full, par);
    static_for<0, SM_C / 64>([&](auto gc) {
      constexpr int G = decltype(gc)::value;
      uint32_t v[32];
      exchange(gc, v);
      const int c0 = G * 64 + half * 32;
      float f[32];
      const float4* b4 = reinterpret_cast<const float4*>(p.b2 + c0);
      uint8_t* row = sX + G * SM_SUB + r * 128;
      const int ch0 = half * 4;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float4 ba = __ldg(b4 + 2 * i), bb = __ldg(b4 + 2 * i + 1);
        uint4* dst = reinterpret_cast<uint4*>(row + (((ch0 + i) ^ (r & 7)) << 4));
        const uint4 u = *dst;
        const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), cc = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
        f[8 * i + 0] = __uint_as_float(v[8 * i + 0]) + ba.x + a.x;  f[8 * i + 1] = __uint_as_float(v[8 * i + 1]) + ba.y + a.y;
        f[8 * i + 2] = __uint_as_float(v[8 * i + 2]) + ba.z + b.x;  f[8 * i + 3] = __uint_as_float(v[8 * i + 3]) + ba.w + b.y;
        f[8 * i + 4] = __uint_as_float(v[8 * i + 4]) + bb.x + cc.x; f[8 * i + 5] = __uint_as_float(v[8 * i + 5]) + bb.y + cc.y;
        f[8 * i + 6] = __uint_as_float(v[8 * i + 6]) + bb.z + d.x;  f[8 * i + 7] = __uint_as_float(v[8 * i + 7]) + bb.w + d.y;
        uint4 o;
        o.x = pack_bf16x2(f[8 * i + 0], f[8 * i + 1]); o.y = pack_bf16x2(f[8 * i + 2], f[8 * i + 3]);
        o.z = pack_bf16x2(f[8 * i + 4], f[8 * i + 5]); o.w = pack_bf16x2(f[8 * i + 6], f[8 * i + 7]);
        *dst = o;
      }
      if (p.gn_stats != nullptr)
        gn_chunk_stats<8>(f, p.gn_stats + (((size_t)tile * 4 + quad) * 32 + c0 / 8) * 2, 0, lane);
    });
    fence_proxy_async();
    mbar_arrive(&bar->out_ready);
  }
}

__global__ void __launch_bounds__(SM_THREADS, 1)
swin_mlp_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmO,
                const __grid_constant__ CUtensorMap tmW1, const __grid_constant__ CUtensorMap tmW2,
                const SwinMlpParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];     // no static smem in this kernel: the window starts 1024-aligned
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  uint8_t* sX = smem;                                   // the tile buffer: 4 sub-tiles of [128 x 64]
  uint8_t* sW = smem + 4 * SM_SUB;                      // weight ring
  float* xacc = reinterpret_cast<float*>(sW + SM_WST * SM_WBYTES);        // [128 rows][SM_XLD]
  float2* xln = reinterpret_cast<float2*>(sW + SM_WST * SM_WBYTES + SM_XCH);   // [128 rows] (sum, sumsq)
  SmBars* bar = reinterpret_cast<SmBars*>(xln + 128);
  uint64_t* w_full = reinterpret_cast<uint64_t*>(bar + 1);               // [SM_WST]
  uint64_t* w_empty = w_full + SM_WST;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmX); tma_prefetch_desc(&tmO); tma_prefetch_desc(&tmW1); tma_prefetch_desc(&tmW2);
    mbar_init(&bar->x_full, 1); mbar_init(&bar->res_full, 1);
    mbar_init(&bar->acc2_done, 8); mbar_init(&bar->out_ready, 256);
    for (int i = 0; i < SM_WST; ++i) { mbar_init(&w_full[i], 1); mbar_init(&w_empty[i], 8); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ------------------------------------------------------------------ weight producer: W1 then W2 per tile
    int st = 0;
    uint32_t ph = 0;
    for (int tile = blockIdx.x; tile < p.m_tiles; tile += gridDim.x) {
      for (int gemm = 0; gemm < 2; ++gemm) {
        for (int kb = 0; kb < 4; ++kb) {
          mbar_wait(&w_empty[st], ph ^ 1);
          if (elect_one()) {
            mbar_arrive_expect_tx(&w_full[st], SM_WBYTES);
            tma_load_2d(sW + st * SM_WBYTES, gemm == 0 ? &tmW1 : &tmW2, &w_full[st], kb * 64, 0);
          }
          __syncwarp();
          if (++st == SM_WST) { st = 0; ph ^= 1; }
        }
      }
    }
  } else if (warp == 9) {
    // ------------------------------------------------------------------ DMA warp
    uint32_t par = 0;
    for (int tile = blockIdx.x; tile < p.m_tiles; tile += gridDim.x, par ^= 1) {
      if (lane == 0) {
        mbar_arrive_expect_tx(&bar->x_full, 4 * SM_SUB);
        for (int kb = 0; kb < 4; ++kb) tma_load_2d(sX + kb * SM_SUB, &tmX, &bar->x_full, kb * 64, tile * SM_BM);
      }
      __syncwarp();
      mbar_wait(&bar->acc2_done, par);          // GEMM2 has consumed the buffer: bring x back for the residual
      if (lane == 0) {
        mbar_arrive_expect_tx(&bar->res_full, 4 * SM_SUB);
        for (int kb = 0; kb < 4; ++kb) tma_load_2d(sX + kb * SM_SUB, &tmX, &bar->res_full, kb * 64, tile * SM_BM);
      }
      __syncwarp();
      mbar_wait(&bar->out_ready, par);
      if (lane == 0) {
        for (int kb = 0; kb < 4; ++kb) tma_store_2d(&tmO, sX + kb * SM_SUB, kb * 64, tile * SM_BM);
        bulk_commit();
        bulk_wait_read<0>();          // the buffer may be refilled
      }
      __syncwarp();
    }
    if (lane == 0) bulk_wait0();
  } else {
    swin_mlp_compute(p, sX, sW, xacc, xln, bar, w_full, w_empty, warp, lane);

  }
}

static int enc2d(CUtensorMap* map, const void* base, int ld, long long rows, int cols, int box_rows) {
  return tmap_rows_bf16(map, base, ld, rows, cols, box_rows);
}

}  // namespace pgt

using namespace pgt;

extern "C" int pgt_swin_mlp_bf16(const void* x, int ldx, int T, int C, const float* ln_g, const float* ln_b, float eps,
                                 const void* W1, const float* b1, const void* W2, const float* b2, void* out, int ldo,
                                 float* gn_stats, void* stream) {
  PGT_CHECK_ARG(x && out && W1 && W2 && b1 && b2 && T > 0 && ((ln_g == nullptr) == (ln_b == nullptr)));   // both null: no affine
  if (C != SM_C) return PGT_ERR_UNSUPPORTED;
  auto al = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  PGT_CHECK_ARG(al(x) && al(out) && al(W1) && al(W2) && ldx % 8 == 0 && ldo % 8 == 0);
  CUtensorMap tx, to, t1, t2;
  int rc = enc2d(&tx, x, ldx, T, C, SM_BM);
  if (rc == PGT_OK) rc = enc2d(&to, out, ldo, T, C, SM_BM);
  if (rc == PGT_OK) rc = enc2d(&t1, W1, C, C, C, SM_C);
  if (rc == PGT_OK) rc = enc2d(&t2, W2, C, C, C, SM_C);
  if (rc != PGT_OK) return rc;
  static PerDeviceOnce once;
  PGT_CUDA_OK(once.run([] { return cudaFuncSetAttribute(swin_mlp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SM_SMEM); }));
  SwinMlpParams p{};
  p.T = T; p.m_tiles = ceil_div(T, SM_BM);
  p.ln_g = ln_g; p.ln_b = ln_b; p.eps = eps; p.b1 = b1; p.b2 = b2; p.gn_stats = gn_stats;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int grid = p.m_tiles < num_sms() ? p.m_tiles : num_sms();
  {
    ProfScope ps(PGT_PROF_GEMM, 4.0 * (double)T * C * C, st, "swin_mlp_fused C256");
    swin_mlp_kernel<<<grid, SM_THREADS, SM_SMEM, st>>>(tx, to, t1, t2, p);
  }
  PGT_LAUNCH_OK();
  return PGT_OK;
}
