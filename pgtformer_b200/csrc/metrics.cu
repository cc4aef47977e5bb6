// Full-reference scores of restored frames against ground truth, as the reference's test configuration asks for them
// (options/release_test_stage_IIII_dont_need_align_version.yml, val.metrics: calculate_psnr and calculate_ssim of
// basicsr 1.4 with crop_border 0 and test_y_channel false, over the rgb frame; restated in oracle/metrics_oracle.py).
//   frame_scores_tile_kernel: one CTA per 32 x 32 tile of one frame pair, all three channels.  Both frames' uint8 tile
//     and a 5-pixel halo go to shared memory; per channel, a horizontal 11-tap pass writes the five filtered fields of
//     x, y, x^2, y^2 and xy for the tile's 42 rows to shared memory in fp64, and a vertical pass finishes them in
//     registers and evaluates the SSIM map at the tile's pixels of the valid region [5, H - 5) x [5, W - 5).  The CTA
//     also sums (a - b)^2 over its 32 x 32 x 3 values exactly, in integers.  Per-CTA partials go to the workspace.
//   frame_scores_finish_kernel: one CTA per frame sums its tiles' partials in a fixed order: sse, and each channel's
//     map mean.
// No floating-point atomics: every sum has a fixed order, so a call gives the same bits on every run.
#include <cmath>

#include "common.cuh"
#include "tmap.cuh"

namespace pgt {

constexpr int FS_T = 32;                    // output tile side
constexpr int FS_R = 5;                     // window radius (11 taps)
constexpr int FS_S = FS_T + 2 * FS_R;       // tile side with the halo
constexpr int FS_THREADS = 256;
constexpr int FS_COLS = 4;                  // consecutive columns per item of the horizontal pass
constexpr int FS_ROWS = FS_T * FS_T / FS_THREADS;   // consecutive rows per thread of the vertical pass
constexpr int FS_PART = 4;                  // workspace doubles per tile: three channel map sums, sse (uint64 bits)
constexpr int FS_FIN_THREADS = 128;
constexpr int FS_TILE_BYTES = (FS_S * FS_S * 3 + 15) / 16 * 16;
constexpr int FS_SMEM = 2 * FS_TILE_BYTES + 5 * FS_S * FS_T * (int)sizeof(double);

// The Gaussian window cv2.getGaussianKernel(11, 1.5) returns: exp(-(i - 5)^2 / (2 1.5^2)), normalised to sum 1.
// Passed by value, so a launch needs no constant upload and stays capture-safe.
struct FsWindow {
  double k[2 * FS_R + 1];
};

// Exact uint32 -> fp64 on the FP64 pipe: v in the low mantissa bits of 2^52, minus 2^52.  The horizontal pass
// converts five integer sums per tap pair, which would otherwise queue on the slower conversion unit.
__device__ __forceinline__ double u2d(uint32_t v) { return __hiloint2double(0x43300000, (int)v) - 4503599627370496.0; }

__device__ __forceinline__ double block_sum_fixed(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double s = 0.0;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += red[w];
  return s;
}

__global__ void __launch_bounds__(FS_THREADS)
frame_scores_tile_kernel(const uint8_t* __restrict__ a, const uint8_t* __restrict__ b, int H, int W, int tiles_x,
                         int tiles, const FsWindow win, double* __restrict__ ws) {
  extern __shared__ __align__(16) unsigned char fs_smem[];
  uint8_t* ta = fs_smem;
  uint8_t* tb = fs_smem + FS_TILE_BYTES;
  double* hs = reinterpret_cast<double*>(fs_smem + 2 * FS_TILE_BYTES);   // [5][FS_S][FS_T]
  __shared__ double red[FS_THREADS / 32];
  __shared__ unsigned long long red_sse[FS_THREADS / 32];

  const int f = blockIdx.x / tiles, t = blockIdx.x - f * tiles;
  const int r0 = (t / tiles_x) * FS_T, c0 = (t - (t / tiles_x) * tiles_x) * FS_T;
  const size_t frame = (size_t)H * W * 3;
  const uint8_t* fa = a + f * frame;
  const uint8_t* fb = b + f * frame;

  // the tile and its halo, zero outside the frame (those values reach no output of the valid region)
  for (int i = threadIdx.x; i < FS_S * FS_S * 3; i += FS_THREADS) {
    const int r = i / (FS_S * 3), q = i - r * (FS_S * 3);
    const int gr = r0 - FS_R + r, gq = (c0 - FS_R) * 3 + q;
    const bool in = gr >= 0 && gr < H && gq >= 0 && gq < W * 3;
    const size_t off = (size_t)gr * W * 3 + gq;
    ta[i] = in ? __ldg(fa + off) : 0;
    tb[i] = in ? __ldg(fb + off) : 0;
  }
  __syncthreads();

  // sse over the tile's own pixels, exact: at most 12 squares of <= 255^2 per thread
  uint32_t sq = 0;
  for (int i = threadIdx.x; i < FS_T * FS_T * 3; i += FS_THREADS) {
    const int r = i / (FS_T * 3), q = i - r * (FS_T * 3);
    if (r0 + r < H && c0 * 3 + q < W * 3) {
      const int s = FS_R + r, p = s * FS_S * 3 + FS_R * 3 + q;
      const int d = (int)ta[p] - (int)tb[p];
      sq += (uint32_t)(d * d);
    }
  }

  const int vj = threadIdx.x & (FS_T - 1), vi0 = (threadIdx.x / FS_T) * FS_ROWS;
  double* out = ws + (size_t)blockIdx.x * FS_PART;
  for (int c = 0; c < 3; ++c) {
    // horizontal pass: items (row, 4 columns); the symmetric window pairs taps q and 10 - q, whose integer sums
    // are exact, so each field takes 6 conversions and 6 fma per output instead of 11 of each
    for (int it = threadIdx.x; it < FS_S * (FS_T / FS_COLS); it += FS_THREADS) {
      const int r = it / (FS_T / FS_COLS), j0 = (it - r * (FS_T / FS_COLS)) * FS_COLS;
      const uint8_t* ra = ta + r * FS_S * 3 + j0 * 3 + c;
      const uint8_t* rb = tb + r * FS_S * 3 + j0 * 3 + c;
      uint32_t x[FS_COLS + 2 * FS_R], y[FS_COLS + 2 * FS_R];
#pragma unroll
      for (int q = 0; q < FS_COLS + 2 * FS_R; ++q) {
        x[q] = ra[3 * q];
        y[q] = rb[3 * q];
      }
#pragma unroll
      for (int m = 0; m < FS_COLS; ++m) {
        double sx = 0.0, sy = 0.0, sxx = 0.0, syy = 0.0, sxy = 0.0;
#pragma unroll
        for (int q = 0; q <= FS_R; ++q) {
          const uint32_t x0 = x[m + q], y0 = y[m + q];
          const uint32_t x1 = q < FS_R ? x[m + 2 * FS_R - q] : 0u, y1 = q < FS_R ? y[m + 2 * FS_R - q] : 0u;
          const double k = win.k[q];
          sx = fma(k, u2d(x0 + x1), sx);
          sy = fma(k, u2d(y0 + y1), sy);
          sxx = fma(k, u2d(x0 * x0 + x1 * x1), sxx);
          syy = fma(k, u2d(y0 * y0 + y1 * y1), syy);
          sxy = fma(k, u2d(x0 * y0 + x1 * y1), sxy);
        }
        double* h = hs + r * FS_T + j0 + m;
        h[0 * FS_S * FS_T] = sx;
        h[1 * FS_S * FS_T] = sy;
        h[2 * FS_S * FS_T] = sxx;
        h[3 * FS_S * FS_T] = syy;
        h[4 * FS_S * FS_T] = sxy;
      }
    }
    __syncthreads();

    // vertical pass: column vj, rows vi0 .. vi0 + 3, each field row read once for the four outputs
    double v[5][FS_ROWS];
#pragma unroll
    for (int e = 0; e < 5; ++e)
#pragma unroll
      for (int o = 0; o < FS_ROWS; ++o) v[e][o] = 0.0;
#pragma unroll
    for (int r = 0; r < FS_ROWS + 2 * FS_R; ++r) {
#pragma unroll
      for (int e = 0; e < 5; ++e) {
        const double hv = hs[(e * FS_S + vi0 + r) * FS_T + vj];
#pragma unroll
        for (int o = 0; o < FS_ROWS; ++o)
          if (r - o >= 0 && r - o <= 2 * FS_R) v[e][o] = fma(win.k[r - o], hv, v[e][o]);
      }
    }
    // the map, with one rounding per operation as numpy forms it: identical frames give exactly 1
    const double C1 = (0.01 * 255.0) * (0.01 * 255.0), C2 = (0.03 * 255.0) * (0.03 * 255.0);
    double s = 0.0;
#pragma unroll
    for (int o = 0; o < FS_ROWS; ++o) {
      const int gi = r0 + vi0 + o, gj = c0 + vj;
      if (gi >= FS_R && gi < H - FS_R && gj >= FS_R && gj < W - FS_R) {
        const double mu1 = v[0][o], mu2 = v[1][o];
        const double mu1_sq = __dmul_rn(mu1, mu1), mu2_sq = __dmul_rn(mu2, mu2), mu1_mu2 = __dmul_rn(mu1, mu2);
        const double s1 = __dsub_rn(v[2][o], mu1_sq), s2 = __dsub_rn(v[3][o], mu2_sq), s12 = __dsub_rn(v[4][o], mu1_mu2);
        const double num = __dmul_rn(__dadd_rn(__dmul_rn(2.0, mu1_mu2), C1), __dadd_rn(__dmul_rn(2.0, s12), C2));
        const double den = __dmul_rn(__dadd_rn(__dadd_rn(mu1_sq, mu2_sq), C1), __dadd_rn(__dadd_rn(s1, s2), C2));
        s += __ddiv_rn(num, den);
      }
    }
    s = block_sum_fixed(s, red);                             // its first barrier also frees hs for the next channel
    if (threadIdx.x == 0) out[c] = s;
  }
  unsigned long long q = sq;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  if ((threadIdx.x & 31) == 0) red_sse[threadIdx.x >> 5] = q;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long s = 0;
    for (int w = 0; w < FS_THREADS / 32; ++w) s += red_sse[w];
    reinterpret_cast<unsigned long long*>(out)[3] = s;
  }
}

__global__ void __launch_bounds__(FS_FIN_THREADS)
frame_scores_finish_kernel(const double* __restrict__ ws, int tiles, double valid, unsigned long long* __restrict__ sse,
                           double* __restrict__ ssim) {
  __shared__ double red[FS_FIN_THREADS / 32];
  __shared__ unsigned long long red_sse[FS_FIN_THREADS / 32];
  const int f = blockIdx.x;
  const double* p = ws + (size_t)f * tiles * FS_PART;
  double s[3] = {0.0, 0.0, 0.0};
  unsigned long long q = 0;
  for (int t = threadIdx.x; t < tiles; t += FS_FIN_THREADS) {
#pragma unroll
    for (int c = 0; c < 3; ++c) s[c] += p[(size_t)t * FS_PART + c];
    q += reinterpret_cast<const unsigned long long*>(p)[(size_t)t * FS_PART + 3];
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const double m = block_sum_fixed(s[c], red);
    if (threadIdx.x == 0) ssim[3 * f + c] = m / valid;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  if ((threadIdx.x & 31) == 0) red_sse[threadIdx.x >> 5] = q;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long t = 0;
    for (int w = 0; w < FS_FIN_THREADS / 32; ++w) t += red_sse[w];
    sse[f] = t;
  }
}

static long long fs_tiles(int H, int W) { return (long long)((H + FS_T - 1) / FS_T) * ((W + FS_T - 1) / FS_T); }

}  // namespace pgt

using namespace pgt;

extern "C" long long pgt_frame_scores_ws_doubles(int F, int H, int W) {
  return F > 0 && H > 0 && W > 0 ? (long long)F * fs_tiles(H, W) * FS_PART : 0;
}

extern "C" int pgt_frame_scores(const void* a_u8, const void* b_u8, int F, int H, int W, double* ws, uint64_t* sse,
                                double* ssim, void* stream) {
  PGT_CHECK_ARG(a_u8 && b_u8 && ws && sse && ssim && F > 0 && H >= 2 * FS_R + 1 && W >= 2 * FS_R + 1);
  PGT_CHECK_ARG((long long)F * fs_tiles(H, W) <= 0x7fffffffLL && (long long)W * 3 <= 0x7fffffffLL);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  static PerDeviceOnce once;                                 // 63 KB of dynamic shared memory: above the default limit
  PGT_CUDA_OK(once.run([] {
    return cudaFuncSetAttribute(frame_scores_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FS_SMEM);
  }));
  FsWindow win;
  double sum = 0.0;
  for (int i = 0; i <= 2 * FS_R; ++i) {
    const double d = i - FS_R;
    win.k[i] = std::exp(-d * d / (2.0 * 1.5 * 1.5));
    sum += win.k[i];
  }
  for (int i = 0; i <= 2 * FS_R; ++i) win.k[i] /= sum;
  const int tiles_x = (W + FS_T - 1) / FS_T, tiles = (int)fs_tiles(H, W);
  {
    ProfScope ps(PGT_PROF_MOVE, 6.0 * F * (double)H * W, st, "pgt_frame_scores");
    frame_scores_tile_kernel<<<F * tiles, FS_THREADS, FS_SMEM, st>>>(
        static_cast<const uint8_t*>(a_u8), static_cast<const uint8_t*>(b_u8), H, W, tiles_x, tiles, win, ws);
    PGT_LAUNCH_OK();
  }
  {
    ProfScope ps(PGT_PROF_MOVE, 32.0 * F * tiles, st, "pgt_frame_scores_finish");
    frame_scores_finish_kernel<<<F, FS_FIN_THREADS, 0, st>>>(ws, tiles, (double)(H - 2 * FS_R) * (W - 2 * FS_R),
                                                             reinterpret_cast<unsigned long long*>(sse), ssim);
    PGT_LAUNCH_OK();
  }
  return PGT_OK;
}
