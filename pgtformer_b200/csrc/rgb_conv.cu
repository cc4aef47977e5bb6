// The two Cin = 3 convolutions on wgmma: Encoder.conv_in (3x3 / 1, archs/tdcrqvae3_arch.py:500-504) and the BiSeNet
// stem Resnet18.conv1 + bn1 + relu (7x7 / 2, archs/pgtformer_arch.py:95-99,110-112) read the fp32 NCHW image directly.
// K = 27 / 147 is far too small for a TMA-fed implicit GEMM (no 16-byte channel vectors to tile), and a patch matrix
// in HBM costs more than the conv, so the im2col happens inside the kernel:
//
//   builders     (4 warps for 3x3, 8 for 7x7: two threads share a pixel, each gathers half of its K range): thread = one
//                output pixel; gathers its 3 k^2 inputs (coalesced across the warp: lanes are neighbouring pixels),
//                optional (x - mean) / std, bf16, and writes the row of the 128 x K A tile straight into the
//                128B-swizzled K-major layout the wgmma descriptor expects (double buffered)
//   last 4 warps one warpgroup: 2 x K/16 wgmma 64 x N x 16 per tile (both 64-row halves) against the weight tile
//                resident in smem, [128 x N] fp32 accumulator in registers -> shared-memory exchange (thread = row)
//                -> bias (+ReLU) -> optional GroupNorm(32) partial statistics -> bf16 -> swizzled staging tile -> one
//                TMA store per 64-channel panel
// N = 64 output channels for both layers; the 3x3 stem also has N = 128 (ch = 128 RQ-VAEs, archs/rqvae_arch.py:592-596).
// The 3x3 N = 64 kernel runs two CTAs per SM (109 KB of shared memory each): a tile's chain gather -> MMA -> epilogue ->
// store is latency-bound, a second CTA fills the gaps.  At N = 128 the staging tiles and the fp32 exchange double
// (179 KB), so one CTA per SM: two would need a single-buffered staging tile and a half-width exchange, i.e. a second
// barrier round per tile, for a layer that is ~1 % of an RQ-VAE forward.
#include <cudaTypedefs.h>

#include "common.cuh"
#include "tmap.cuh"
#include "ptx.cuh"
#include "epi_common.cuh"

namespace pgt {

constexpr int RC_SUB = 128 * 128;        // [128 rows x 64 k] bf16 A sub-tile; also one 64-channel staging panel

struct RgbConvParams {
  const float* x;                        // [F, 3, H, W] fp32
  int H, W, Ho, Wo;
  long long M;                           // F * Ho * Wo output pixels
  int m_tiles;
  float mean[3], istd[3];
  const float* bias;
  int relu;
  float* gn_stats;                       // optional [m_tiles][4][32][2]
};

template <int KS, int N>
struct RgbCfg {
  static_assert(N == 64 || N == 128, "output channels");
  static constexpr int K = 3 * KS * KS;
  static constexpr int KSTEPS = (K + 15) / 16;
  static constexpr int NSUB = (KSTEPS + 3) / 4;
  static constexpr int NCH = KSTEPS * 2;                        // 16-byte chunks written per row
  static constexpr int BSUB = N * 128;                          // [N rows x 64 k] bf16 weight sub-tile
  static constexpr int PANELS = N / 64;                         // 64-channel panels of a staged output tile
  static constexpr int XLD = N + 4;                             // accumulator exchange pitch (fp32)
  static constexpr int XCH = 128 * XLD * 4;
  static constexpr int A_BYTES = NSUB * RC_SUB;
  static constexpr int B_BYTES = NSUB * BSUB;
  static constexpr int STG = PANELS * RC_SUB;                   // one staging tile
  static constexpr int SMEM = 2 * A_BYTES + B_BYTES + 2 * STG + XCH + 256;
  static constexpr int BW = KS == 3 ? 4 : 8;                    // builder warps
  static constexpr int PARTS = BW / 4;                          // threads per output pixel
  static constexpr int THREADS = (BW + 4) * 32;
  static constexpr int PER_SM = KS == 3 && N == 64 ? 2 : 1;     // resident CTAs per SM
};

// 16-byte chunks [CH0, CH1) of one A row (one output pixel): every tap offset is a compile-time constant
template <int KS, int CH0, int CH1>
__device__ __forceinline__ void rgb_build_chunks(const RgbConvParams& p, const float* x0, size_t plane, int iy0, int ix0, bool valid,
                                                 uint8_t* arow, int r) {
  constexpr int K = 3 * KS * KS;
#pragma unroll
  for (int ch = CH0; ch < CH1; ++ch) {
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int k = ch * 8 + j;
      if (k < K) {
        const int tap = k / 3, c = k - tap * 3;
        const int ky = tap / KS, kx = tap - ky * KS;
        const bool ok = valid && (unsigned)(iy0 + ky) < (unsigned)p.H && (unsigned)(ix0 + kx) < (unsigned)p.W;
        v[j] = ok ? (__ldg(x0 + c * plane + ky * p.W + kx) - p.mean[c]) * p.istd[c] : 0.f;
      } else {
        v[j] = 0.f;
      }
    }
    uint4 u;
    u.x = pack_bf16x2(v[0], v[1]); u.y = pack_bf16x2(v[2], v[3]);
    u.z = pack_bf16x2(v[4], v[5]); u.w = pack_bf16x2(v[6], v[7]);
    *reinterpret_cast<uint4*>(arow + (ch >> 3) * RC_SUB + (((ch & 7) ^ (r & 7)) << 4)) = u;
  }
}

// BIAS4: the bias is 16-byte aligned and read as float4 (every caller's own bias tensor); otherwise one float at a time
// (a view such as b[1:]), in an instantiation of its own so that the aligned kernel is the same code as without it.
template <int KS, int STRIDE, int PAD, int N, bool BIAS4>
__global__ void __launch_bounds__(RgbCfg<KS, N>::THREADS, RgbCfg<KS, N>::PER_SM)
rgb_conv_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmO, const RgbConvParams p) {
  using Cfg = RgbCfg<KS, N>;
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  uint8_t* sA = smem;                                   // [2][NSUB] sub-tiles
  uint8_t* sB = sA + 2 * Cfg::A_BYTES;                  // [NSUB] weight sub-tiles
  uint8_t* sO = sB + Cfg::B_BYTES;                      // [2] staging tiles
  float* xch = reinterpret_cast<float*>(sO + 2 * Cfg::STG);
  uint64_t* bars = reinterpret_cast<uint64_t*>(sO + 2 * Cfg::STG + Cfg::XCH);
  uint64_t* a_full = bars;           // [2] builders -> MMA warpgroup
  uint64_t* a_free = bars + 2;       // [2] MMA warpgroup (one arrive per warp) -> builders
  uint64_t* b_full = bars + 4;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int BW = Cfg::BW;
  if (warp == BW) {
    if (lane == 0) {
      tma_prefetch_desc(&tmW); tma_prefetch_desc(&tmO);
      for (int i = 0; i < 2; ++i) { mbar_init(&a_full[i], BW * 32); mbar_init(&a_free[i], 4); }
      mbar_init(b_full, 1);
      fence_barrier_init();
      mbar_arrive_expect_tx(b_full, Cfg::B_BYTES);
      for (int s = 0; s < Cfg::NSUB; ++s) tma_load_2d(sB + s * Cfg::BSUB, &tmW, b_full, s * 64, 0);
    }
    __syncwarp();
  }
  __syncthreads();

  if (warp < BW) {
    // ------------------------------------------------------------------ builders
    const int r = threadIdx.x & 127;
    const int part = threadIdx.x >> 7;                  // which share of the row's 16-byte chunks this thread gathers
    constexpr int CH_PER = (Cfg::NCH + Cfg::PARTS - 1) / Cfg::PARTS;
    const size_t plane = (size_t)p.H * p.W;
    const int HoWo = p.Ho * p.Wo;
    int it = 0;
    for (int tile = blockIdx.x; tile < p.m_tiles; tile += gridDim.x, ++it) {
      const int buf = it & 1;
      const long long row = (long long)tile * 128 + r;
      const bool valid = row < p.M;
      const int f = valid ? (int)(row / HoWo) : 0;
      const int rem = valid ? (int)(row - (long long)f * HoWo) : 0;
      const int oy = rem / p.Wo, ox = rem - oy * p.Wo;
      const int iy0 = oy * STRIDE - PAD, ix0 = ox * STRIDE - PAD;
      const float* x0 = p.x + (size_t)f * 3 * plane + (long long)iy0 * p.W + ix0;
      mbar_wait(&a_free[buf], ((it >> 1) & 1) ^ 1);
      uint8_t* arow = sA + buf * Cfg::A_BYTES + r * 128;
      if (part == 0) rgb_build_chunks<KS, 0, CH_PER < Cfg::NCH ? CH_PER : Cfg::NCH>(p, x0, plane, iy0, ix0, valid, arow, r);
      else rgb_build_chunks<KS, CH_PER < Cfg::NCH ? CH_PER : Cfg::NCH, Cfg::NCH>(p, x0, plane, iy0, ix0, valid, arow, r);
      fence_proxy_async();
      mbar_arrive(&a_full[buf]);
    }
  } else {
    // ------------------------------------------------------------------ MMA + epilogue warpgroup
    const int quad = warp & 3;
    const int r = quad * 32 + lane;
    const int et = threadIdx.x - BW * 32;
    const float* xrow = xch + r * Cfg::XLD;
    mbar_wait(b_full, 0);
    int it = 0;
    for (int tile = blockIdx.x; tile < p.m_tiles; tile += gridDim.x, ++it) {
      const int buf = it & 1;
      mbar_wait(&a_full[buf], (it >> 1) & 1);
      float acc0[N / 2], acc1[N / 2];                     // rows [0, 64) and [64, 128) of the tile
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < Cfg::KSTEPS; ++ks) {
        const uint32_t a = smem_u32(sA + buf * Cfg::A_BYTES + (ks >> 2) * RC_SUB);
        const uint64_t db = wgmma_desc_k_sw128(smem_u32(sB + (ks >> 2) * Cfg::BSUB)) + 2 * (ks & 3);
        wgmma_bf16<N>(acc0, wgmma_desc_k_sw128(a) + 2 * (ks & 3), db, ks != 0 ? 1u : 0u);
        wgmma_bf16<N>(acc1, wgmma_desc_k_sw128(a + 64 * 128) + 2 * (ks & 3), db, ks != 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&a_free[buf]);
      // staging[buf] was last read by the store two tiles back; the exchange by the previous tile's epilogue
      if (et == 0) bulk_wait_read<1>();
      named_bar_sync(1, 128);
      acc_to_smem<0, N>(acc0, xch, Cfg::XLD, quad, lane);
      acc_to_smem<0, N>(acc1, xch + 64 * Cfg::XLD, Cfg::XLD, quad, lane);
      named_bar_sync(1, 128);
      uint8_t* srow = sO + buf * Cfg::STG + r * 128;
#pragma unroll
      for (int hb = 0; hb < N / 32; ++hb) {
        uint32_t v[32];
        smem_row_32(xrow + hb * 32, v);
        float f[32];
        if (BIAS4) {
          const float4* b4 = reinterpret_cast<const float4*>(p.bias + hb * 32);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float4 bb = __ldg(b4 + i);
            f[4 * i + 0] = __uint_as_float(v[4 * i + 0]) + bb.x;
            f[4 * i + 1] = __uint_as_float(v[4 * i + 1]) + bb.y;
            f[4 * i + 2] = __uint_as_float(v[4 * i + 2]) + bb.z;
            f[4 * i + 3] = __uint_as_float(v[4 * i + 3]) + bb.w;
          }
        } else {
#pragma unroll
          for (int i = 0; i < 32; ++i) f[i] = __uint_as_float(v[i]) + __ldg(p.bias + hb * 32 + i);
        }
        if (p.relu) {
#pragma unroll
          for (int i = 0; i < 32; ++i) f[i] = fmaxf(f[i], 0.f);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          uint4 o;
          o.x = pack_bf16x2(f[8 * i + 0], f[8 * i + 1]); o.y = pack_bf16x2(f[8 * i + 2], f[8 * i + 3]);
          o.z = pack_bf16x2(f[8 * i + 4], f[8 * i + 5]); o.w = pack_bf16x2(f[8 * i + 6], f[8 * i + 7]);
          *reinterpret_cast<uint4*>(srow + (hb >> 1) * RC_SUB + (((((hb & 1) * 4) + i) ^ (r & 7)) << 4)) = o;
        }
        // GroupNorm(32): N / 32 channels per group, so a 32-column chunk holds 1024 / N groups
        if (p.gn_stats != nullptr)
          gn_chunk_stats<N / 32>(f, p.gn_stats + (((size_t)tile * 4 + quad) * 32 + hb * (1024 / N)) * 2, 0, lane);
      }
      fence_proxy_async();
      named_bar_sync(1, 128);
      if (et == 0) {
#pragma unroll
        for (int pn = 0; pn < Cfg::PANELS; ++pn) tma_store_2d(&tmO, sO + buf * Cfg::STG + pn * RC_SUB, pn * 64, tile * 128);
        bulk_commit();
      }
    }
    if (et == 0) bulk_wait0();
  }
}

static int rc_enc2d(CUtensorMap* map, const void* base, long long ld, long long rows, int cols, int box_rows) {
  return tmap_rows_bf16(map, base, ld, rows, cols, box_rows);
}

template <int KS, int STRIDE, int PAD, int N, bool BIAS4>
static int launch_rgb(const CUtensorMap& tw, const CUtensorMap& to, const RgbConvParams& p, cudaStream_t st, const char* desc) {
  using Cfg = RgbCfg<KS, N>;
  static PerDeviceOnce once;
  PGT_CUDA_OK(once.run([] {
    cudaError_t e = cudaFuncSetAttribute(rgb_conv_kernel<KS, STRIDE, PAD, N, BIAS4>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM);
    if (e != cudaSuccess) return e;
    // the resident-CTA count is fixed by the kernel's own budget (__launch_bounds__, shared memory), not
    // asked of the occupancy calculator: it answered 1 for the 3x3 kernel and left half of every SM idle
    return cudaFuncSetAttribute(rgb_conv_kernel<KS, STRIDE, PAD, N, BIAS4>, cudaFuncAttributePreferredSharedMemoryCarveout,
                                cudaSharedmemCarveoutMaxShared);
  }));
  const int grid = p.m_tiles < num_sms() * Cfg::PER_SM ? p.m_tiles : num_sms() * Cfg::PER_SM;
  {
    ProfScope ps(PGT_PROF_GEMM, 2.0 * (double)p.M * N * Cfg::K, st, desc);
    rgb_conv_kernel<KS, STRIDE, PAD, N, BIAS4><<<grid, Cfg::THREADS, Cfg::SMEM, st>>>(tw, to, p);
  }
  PGT_LAUNCH_OK();
  return PGT_OK;
}

}  // namespace pgt

using namespace pgt;

extern "C" int pgt_conv_rgb_bf16(const float* x_nchw, int F, int H, int W, int ksize, int stride, int pad,
                                 const float* mean3, const float* std3, const void* Wp, int ldw, int Cout,
                                 const float* bias, int act, void* out, int ldo, float* gn_stats, void* stream) {
  PGT_CHECK_ARG(x_nchw && Wp && bias && out && F > 0 && H > 0 && W > 0);
  const bool k3 = ksize == 3 && stride == 1 && pad == 1, k7 = ksize == 7 && stride == 2 && pad == 3;
  if (!((Cout == 64 && (k3 || k7)) || (Cout == 128 && k3))) return PGT_ERR_UNSUPPORTED;
  PGT_CHECK_ARG(act == PGT_ACT_NONE || act == PGT_ACT_RELU);
  auto al = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  PGT_CHECK_ARG(al(Wp) && al(out) && ldw % 8 == 0 && ldo % 8 == 0 && ldw >= 3 * ksize * ksize && ldo >= Cout);
  RgbConvParams p{};
  p.x = x_nchw; p.H = H; p.W = W;
  p.Ho = (H + 2 * pad - ksize) / stride + 1;
  p.Wo = (W + 2 * pad - ksize) / stride + 1;
  PGT_CHECK_ARG(p.Ho > 0 && p.Wo > 0);
  p.M = (long long)F * p.Ho * p.Wo;
  p.m_tiles = (int)((p.M + 127) / 128);
  for (int c = 0; c < 3; ++c) {
    p.mean[c] = mean3 ? mean3[c] : 0.f;
    p.istd[c] = std3 ? 1.f / std3[c] : 1.f;
  }
  p.bias = bias; p.relu = act == PGT_ACT_RELU; p.gn_stats = gn_stats;
  if (gn_stats != nullptr && (p.Ho * p.Wo) % 128 != 0) return PGT_ERR_UNSUPPORTED;   // a tile must not straddle frames
  CUtensorMap tw, to;
  // weight rows beyond K inside the last 64-wide box are zero-filled by TMA
  int rc = rc_enc2d(&tw, Wp, ldw, Cout, 3 * ksize * ksize, Cout);
  if (rc == PGT_OK) rc = rc_enc2d(&to, out, ldo, p.M, Cout, 128);
  if (rc != PGT_OK) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (al(bias)) {
    if (Cout == 128) return launch_rgb<3, 1, 1, 128, true>(tw, to, p, st, "rgb_conv 3x3/1 N128");
    return ksize == 3 ? launch_rgb<3, 1, 1, 64, true>(tw, to, p, st, "rgb_conv 3x3/1 N64")
                      : launch_rgb<7, 2, 3, 64, true>(tw, to, p, st, "rgb_conv 7x7/2 N64");
  }
  if (Cout == 128) return launch_rgb<3, 1, 1, 128, false>(tw, to, p, st, "rgb_conv 3x3/1 N128");
  return ksize == 3 ? launch_rgb<3, 1, 1, 64, false>(tw, to, p, st, "rgb_conv 3x3/1 N64")
                    : launch_rgb<7, 2, 3, 64, false>(tw, to, p, st, "rgb_conv 7x7/2 N64");
}
