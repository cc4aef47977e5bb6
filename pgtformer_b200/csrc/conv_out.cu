// decoder.norm_out -> SiLU -> conv_out (3x3, 64 -> 3 channels, fp32 NCHW result) as ONE wgmma kernel
// (`archs/pgtformer_arch.py:707-710`, `archs/tdcrqvae3_arch.py:700-706`: GroupNorm(32, eps 1e-6), swish, Conv2d).
// The activation is a template parameter: VQGAN's and CodeFormer's generator ends in GroupNorm -> Conv2d with no swish
// (`archs/vqgan_arch.py:329-332`, last_silu=False), the SILU = false instantiation.
//
// Why its own kernel: with Cout = 3 the generic halo conv computes a 64-wide tile for 3 useful columns and stores
// fp32 NCHW through its slow path (2.3 ms per 16 clips of 512^2), after a separate GroupNorm apply pass over the
// largest tensor of the model (0.5 ms, 3.2 GB).  Here:
//   * 8 builder warps read the RAW conv input once (128-bit loads, a pixel's 64 channels = one 128-byte row), apply
//     y = silu(x * a[f,c] + b[f,c]) (GroupNorm folded into per-(frame, channel) affine terms) and write the bf16
//     (16+2) x (8+2)-pixel halo slab straight into the 128B-swizzled layout — the normalised tensor never exists in HBM;
//   * one warpgroup issues, per 16x8-pixel tile, 9 taps x 4 k-steps x 2 row halves of wgmma 64x16x16: tap (dy,dx) is
//     the same slab viewed from row dy*10+dx (SBO = slab pitch, as in the halo conv of gemm_tc.cu), the 9 x 16 x 64
//     weight tile is resident in shared memory; the same warpgroup adds the bias to the register accumulators and
//     stores the 3 planes (fp32 NCHW) straight from them.
// Cin = 128 (the ch = 128 RQ-VAE decoders, archs/rqvae_arch.py:738-743): a pixel is two 128-byte SW128 K-panels, so the
// slab and the weight tile hold two panels each (9 taps x 8 k-steps) and ab is [F][2][128]; at 133 KB of shared memory
// it runs one CTA per SM.  The Cin = 64 instantiations are unchanged.
#include <cstdio>

#include "common.cuh"
#include "ptx.cuh"
#include "tmap.cuh"

namespace pgt {

constexpr int CO_TW = 8, CO_TH = 16;                         // output tile: 16 rows x 8 pixels = 128 GEMM rows
constexpr int CO_SW = CO_TW + 2, CO_SH = CO_TH + 2;          // halo slab
constexpr int CO_PITCH = CO_SW * 128;                        // bytes between slab image rows
constexpr int CO_SLAB = ((CO_SH * CO_PITCH + 1023) / 1024) * 1024;   // 23552
constexpr int CO_NB = 16;                                    // padded Cout (wgmma N)
constexpr int CO_BUILDERS = 256;
constexpr int CO_THREADS = CO_BUILDERS + 128;                // builder warps 0..7, MMA / epilogue warpgroup 8..11
template <int CIN>
struct CoCfg {
  static_assert(CIN == 64 || CIN == 128, "conv_out input channels");
  static constexpr int PANELS = CIN / 64;                    // 128-byte K-panels per pixel
  static constexpr int WBYTES = 9 * PANELS * CO_NB * 128;    // [tap][panel][16 rows][64 ch] bf16, K-major SW128
  static constexpr int SMEM = 2 * PANELS * CO_SLAB + WBYTES + 2 * 128 * 4 + 256 + 1024;
  static constexpr int PER_SM = CIN == 64 ? 2 : 1;
};

// silu(v) = v * sigmoid(v) = h + h * tanh(h), h = v / 2: one MUFU (tanh.approx, rel. error 2^-11, below the bf16 rounding
// of the result) instead of the ex2 + rcp pair — the builders are MUFU-bound
__device__ __forceinline__ float silu_tanh(float v) {
  const float h = 0.5f * v;
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(h));
  return fmaf(h, t, h);
}

struct ConvOutParams {
  const __nv_bfloat16* x;      // [F, H, W, 64] raw (pre-norm) input, pixel pitch ldx elements
  int ldx, F, H, W, cout;
  const float* ab;             // [F][2][Cin]
  const __nv_bfloat16* w;      // [cout][9 * Cin] packed (tap-major), row pitch ldw
  int ldw;
  const float* bias;           // [cout] or null
  float* out;                  // [F, cout, H, W]
  int tiles_x, tiles_y, num_tiles;
};

template <bool SILU, int CIN>
__global__ void __launch_bounds__(CO_THREADS, CoCfg<CIN>::PER_SM)
conv_out_gn_kernel(const ConvOutParams p) {
  using Cfg = CoCfg<CIN>;
  constexpr int NP = Cfg::PANELS;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* slab = smem;                                         // [2][NP][CO_SLAB]
  uint8_t* sW = smem + 2 * NP * CO_SLAB;                        // [9][NP][16 x 128 B]
  float* sAB = reinterpret_cast<float*>(sW + Cfg::WBYTES);      // [2][2][64]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sAB + 2 * 128);
  uint64_t* slab_full = bars;                                   // [2] builders -> MMA warpgroup
  uint64_t* slab_empty = bars + 2;                              // [2] MMA warpgroup (one arrive per warp) -> builders

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < 2; ++i) {
      mbar_init(&slab_full[i], CO_BUILDERS);
      mbar_init(&slab_empty[i], 4);
    }
    fence_barrier_init();
  }
  // weights -> swizzled K-major tiles (rows >= cout are zero)
  for (int i = threadIdx.x; i < 9 * NP * CO_NB * 8; i += CO_THREADS) {
    const int tp = i / (CO_NB * 8), r = (i / 8) % CO_NB, ch = i % 8;          // tp = tap * NP + panel
    uint4 v = make_uint4(0, 0, 0, 0);
    if (r < p.cout) v = __ldg(reinterpret_cast<const uint4*>(p.w + (size_t)r * p.ldw + tp * 64 + ch * 8));
    *reinterpret_cast<uint4*>(sW + tp * (CO_NB * 128) + r * 128 + ((ch ^ (r & 7)) << 4)) = v;
  }
  fence_proxy_async();
  __syncthreads();
  const int per_frame = p.tiles_x * p.tiles_y;

  if (warp < CO_BUILDERS / 32) {
    // ------------------------------------------------------------------ slab builders (GroupNorm + SiLU on the way in)
    const int bt = threadIdx.x;                                  // 0..255
    const int chunk = bt & 7;                                    // 8 channels = one 16-byte chunk
    int it = 0;
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x, ++it) {
      const int buf = it & 1;
      const uint32_t ph = (it >> 1) & 1;
      const int f = tile / per_frame, r = tile - f * per_frame;
      const int y0 = (r / p.tiles_x) * CO_TH - 1, x0 = (r % p.tiles_x) * CO_TW - 1;
#pragma unroll
      for (int pn = 0; pn < NP; ++pn) {
      float a[8], b[8];
      {
        const float4* pa = reinterpret_cast<const float4*>(p.ab + (size_t)f * 2 * CIN + pn * 64 + chunk * 8);
        const float4 a0 = __ldg(pa), a1 = __ldg(pa + 1), b0 = __ldg(pa + CIN / 4), b1 = __ldg(pa + CIN / 4 + 1);
        a[0] = a0.x; a[1] = a0.y; a[2] = a0.z; a[3] = a0.w; a[4] = a1.x; a[5] = a1.y; a[6] = a1.z; a[7] = a1.w;
        b[0] = b0.x; b[1] = b0.y; b[2] = b0.z; b[3] = b0.w; b[4] = b1.x; b[5] = b1.y; b[6] = b1.z; b[7] = b1.w;
      }
      // loads first (6 independent 128-bit requests per thread), then wait for the slab, then transform + store
      constexpr int NPIX = CO_SH * CO_SW;                        // 180
      constexpr int ITERS = (NPIX * 8 + CO_BUILDERS - 1) / CO_BUILDERS;   // 6
      uint4 raw[ITERS];
      bool inside[ITERS];
#pragma unroll
      for (int i = 0; i < ITERS; ++i) {
        const int pix = (bt >> 3) + i * (CO_BUILDERS / 8);
        const int sy = pix / CO_SW, sx = pix - sy * CO_SW;
        const int y = y0 + sy, x = x0 + sx;
        inside[i] = pix < NPIX && y >= 0 && y < p.H && x >= 0 && x < p.W;
        raw[i] = make_uint4(0, 0, 0, 0);
        if (inside[i]) raw[i] = __ldg(reinterpret_cast<const uint4*>(p.x + ((size_t)(f * p.H + y) * p.W + x) * p.ldx + pn * 64 + chunk * 8));
      }
      if (pn == 0) mbar_wait(&slab_empty[buf], ph ^ 1);
      uint8_t* sl = slab + (buf * NP + pn) * CO_SLAB;
#pragma unroll
      for (int i = 0; i < ITERS; ++i) {
        const int pix = (bt >> 3) + i * (CO_BUILDERS / 8);
        if (pix < NPIX) {
          uint4 o = make_uint4(0, 0, 0, 0);                      // zero padding applies to the activated tensor
          if (inside[i]) {
            const uint32_t u[4] = {raw[i].x, raw[i].y, raw[i].z, raw[i].w};
            uint32_t q[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const float2 xv = unpack_bf16x2(u[e]);
              const float v0 = fmaf(xv.x, a[2 * e], b[2 * e]), v1 = fmaf(xv.y, a[2 * e + 1], b[2 * e + 1]);
              q[e] = SILU ? pack_bf16x2(silu_tanh(v0), silu_tanh(v1)) : pack_bf16x2(v0, v1);
            }
            o = make_uint4(q[0], q[1], q[2], q[3]);
          }
          *reinterpret_cast<uint4*>(sl + pix * 128 + ((chunk ^ (pix & 7)) << 4)) = o;
        }
      }
      }
      fence_proxy_async();
      mbar_arrive(&slab_full[buf]);
    }
  } else {
    // ------------------------------------------------------------------ MMA warpgroup: wgmma -> + bias -> fp32 NCHW planes
    // Accumulator fragment (m64n16): lane holds columns 2 (lane % 4) + {0, 1} of rows 16 w + lane / 4 (+ 8) of each
    // 64-row half; the lanes with lane % 4 < 2 hold the (at most) three real output channels.
    const int w = warp & 3;
    const int t4 = lane & 3;
    float bias[3] = {0.f, 0.f, 0.f};
    for (int c = 0; c < p.cout && c < 3; ++c) bias[c] = p.bias ? __ldg(p.bias + c) : 0.f;
    const size_t plane = (size_t)p.H * p.W;
    const uint32_t sw = smem_u32(sW);
    int it = 0;
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x, ++it) {
      const int buf = it & 1;
      const uint32_t ph = (it >> 1) & 1;
      const int f = tile / per_frame, r = tile - f * per_frame;
      mbar_wait(&slab_full[buf], ph);
      float acc[2][CO_NB / 2];                                  // tile rows [0, 64) = image rows 0..7, [64, 128) = 8..15
      wgmma_fence();
#pragma unroll
      for (int tap = 0; tap < 9; ++tap) {
#pragma unroll
        for (int pn = 0; pn < NP; ++pn) {
        const uint32_t sa = smem_u32(slab + (buf * NP + pn) * CO_SLAB);
        const uint32_t ta = sa + ((tap / 3) * CO_SW + (tap % 3)) * 128;
        const uint64_t da0 = wgmma_desc_k_sw128(ta, CO_PITCH), da1 = wgmma_desc_k_sw128(ta + 8 * CO_PITCH, CO_PITCH);
        const uint64_t db = wgmma_desc_k_sw128(sw + (tap * NP + pn) * (CO_NB * 128));
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          wgmma_bf16<CO_NB>(acc[0], da0 + 2 * k, db + 2 * k, (tap | pn | k) != 0 ? 1u : 0u);
          wgmma_bf16<CO_NB>(acc[1], da1 + 2 * k, db + 2 * k, (tap | pn | k) != 0 ? 1u : 0u);
        }
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&slab_empty[buf]);
      if (t4 < 2) {
        float* o = p.out + (size_t)f * p.cout * plane;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int row = 64 * h + 16 * w + (lane >> 2) + 8 * (e >> 1);   // GEMM row = pixel (ty = row / 8, tx = row % 8)
            const int c = 2 * t4 + (e & 1);
            const int y = (r / p.tiles_x) * CO_TH + (row >> 3), x = (r % p.tiles_x) * CO_TW + (row & 7);
            if (c < p.cout) o[c * plane + (size_t)y * p.W + x] = acc[h][e] + bias[c < 3 ? c : 0];
          }
        }
      }
    }
  }
}

}  // namespace pgt

using namespace pgt;

template <bool SILU, int CIN>
static int conv_out_gn_launch(const ConvOutParams& p, int Cin, cudaStream_t st) {
  using Cfg = CoCfg<CIN>;
  static PerDeviceOnce once;
  PGT_CUDA_OK(once.run([] { return cudaFuncSetAttribute(conv_out_gn_kernel<SILU, CIN>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM); }));
  // Cin = 64: 2 CTAs per SM (66 KB smem each); Cin = 128: one (133 KB)
  const int grid = p.num_tiles < Cfg::PER_SM * num_sms() ? p.num_tiles : Cfg::PER_SM * num_sms();
  char desc[64];
  snprintf(desc, sizeof(desc), "conv_out_gn%s F%d H%d W%d N%d", SILU ? "" : "_nosilu", p.F, p.H, p.W, p.cout);
  ProfScope ps(PGT_PROF_GEMM, 2.0 * p.F * (double)p.H * p.W * p.cout * 9 * Cin, st, desc);
  conv_out_gn_kernel<SILU, CIN><<<grid, CO_THREADS, Cfg::SMEM, st>>>(p);
  PGT_LAUNCH_OK();
  return PGT_OK;
}

template <bool SILU>
static int conv_out_gn_run(const void* x, int F, int H, int W, int Cin, int ldx, const float* gn_ab, const void* Wp, int ldw,
                           int Cout, const float* bias, float* out, void* stream) {
  PGT_CHECK_ARG(x && gn_ab && Wp && out && F > 0);
  if ((Cin != 64 && Cin != 128) || Cout < 1 || Cout > 3 || H % CO_TH != 0 || W % CO_TW != 0 || ldx % 8 != 0 || ldw % 8 != 0)
    return PGT_ERR_UNSUPPORTED;
  PGT_CHECK_ARG((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(Wp) & 15) == 0 &&
                (reinterpret_cast<uintptr_t>(gn_ab) & 15) == 0);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ConvOutParams p{};
  p.x = reinterpret_cast<const __nv_bfloat16*>(x); p.ldx = ldx; p.F = F; p.H = H; p.W = W; p.cout = Cout;
  p.ab = gn_ab; p.w = reinterpret_cast<const __nv_bfloat16*>(Wp); p.ldw = ldw; p.bias = bias; p.out = out;
  p.tiles_x = W / CO_TW; p.tiles_y = H / CO_TH; p.num_tiles = F * p.tiles_x * p.tiles_y;
  return Cin == 64 ? conv_out_gn_launch<SILU, 64>(p, Cin, st) : conv_out_gn_launch<SILU, 128>(p, Cin, st);
}

extern "C" int pgt_conv_out_gn(const void* x, int F, int H, int W, int Cin, int ldx, const float* gn_ab, const void* Wp,
                               int ldw, int Cout, const float* bias, float* out, void* stream) {
  return conv_out_gn_run<true>(x, F, H, W, Cin, ldx, gn_ab, Wp, ldw, Cout, bias, out, stream);
}

extern "C" int pgt_conv_out_gn_act(const void* x, int F, int H, int W, int Cin, int ldx, const float* gn_ab, const void* Wp,
                                   int ldw, int Cout, const float* bias, float* out, int silu, void* stream) {
  PGT_CHECK_ARG(silu == 0 || silu == 1);
  return silu ? conv_out_gn_run<true>(x, F, H, W, Cin, ldx, gn_ab, Wp, ldw, Cout, bias, out, stream)
              : conv_out_gn_run<false>(x, F, H, W, Cin, ldx, gn_ab, Wp, ldw, Cout, bias, out, stream);
}
