// The `lr` degradation of the reference's test set: basicsr's antialiased bicubic imresize (matlab_functions.py,
// restated in oracle/degrade_oracle.py) of rgb24 frames, (float)(v / 255.0) in, fp32 planes out, both passes in one
// launch.  Each output value of a pass is defined as the fp32 value nearest to the exact sum of its fp32 products
// w * x (ties to even), so it does not depend on any summation order: tiling, batch size and graph replay give the
// same bits.
//   imresize_kernel: one CTA per (frame, TH x TW output tile).  The tile's source footprint (a contiguous block of
//     rows and columns: the tap indices are mirrored into the frame by the table's builder, and a mirrored tile's
//     indices still span no more than its unmirrored ones) goes to shared memory as uint8; the H pass writes the
//     tile's TH rows over the footprint's columns to shared memory in fp32 (basicsr's out_1), and the W pass reads
//     them from there.
// The tap tables (weights fp32 [out, K], indices int32 [out, K] in [0, in)) are built and checked by
// pgtformer_b200/degrade.py, the only builder; DESIGN.md §6d gives the exactness argument the builder checks.
#include <algorithm>

#include "common.cuh"
#include "tmap.cuh"

namespace pgt {

constexpr int DG_THREADS = 256;
constexpr int DG_SMEM_MAX = 112 * 1024;      // tiles are shrunk until their footprint fits

// Sum of fp64 terms, each an exact fp32 x fp32 product, kept exactly as hi + lo (TwoSum of each term into hi, the
// rounding errors summed in lo: exact while |lo| stays below 2^53 times the terms' common quantum, which the table
// builder checks), then rounded once to fp32: TwoSum(hi, lo) = s + t exactly, s made round-to-odd at 53 bits from t's
// sign, and round-to-odd at 53 bits followed by one rounding to 24 bits is the correctly rounded fp32 value.
struct ExactSum {
  double hi = 0.0, lo = 0.0;
  __device__ __forceinline__ void add(float w, float x) {
    const double p = __dmul_rn((double)w, (double)x);
    const double s = __dadd_rn(hi, p);
    const double bp = __dsub_rn(s, hi);
    const double e = __dadd_rn(__dsub_rn(hi, __dsub_rn(s, bp)), __dsub_rn(p, bp));
    hi = s;
    lo = __dadd_rn(lo, e);
  }
  __device__ __forceinline__ float value() const {
    const double s = __dadd_rn(hi, lo);
    const double bp = __dsub_rn(s, hi);
    const double t = __dadd_rn(__dsub_rn(hi, __dsub_rn(s, bp)), __dsub_rn(lo, bp));
    long long b = __double_as_longlong(s);
    if (t != 0.0 && (b & 1) == 0) b += ((t > 0.0) == (s > 0.0)) ? 1 : -1;     // one step toward t: round to odd
    return __double2float_rn(__longlong_as_double(b));
  }
};

// Footprint side (rows or columns) of T consecutive outputs of a K-tap table over an axis of n samples.  basicsr's
// taps for scale s are ceil(4 / s) + 2 minus at most the two trimmed columns, so 1 / s <= K / 4; consecutive outputs
// are 1 / s apart, so T of them span at most (T - 1) K / 4 + 1 + K unmirrored samples, and mirroring only folds them.
__host__ __device__ __forceinline__ int dg_span(int T, int K, int n) {
  return std::min(n, ((T - 1) * K + 3) / 4 + K + 2);
}

static size_t dg_smem(int TH, int TW, int Kh, int Kw, int h, int w) {
  const size_t rows = dg_span(TH, Kh, h), cols = dg_span(TW, Kw, w);
  return (size_t)(TH * Kh + TW * Kw) * 8 + 256 * 4 + (rows * cols * 3 + 15) / 16 * 16 + 3 * (size_t)TH * cols * 4;
}

__global__ void __launch_bounds__(DG_THREADS)
imresize_kernel(const uint8_t* __restrict__ x, int h, int w, const float* __restrict__ wts_h,
                const int* __restrict__ idx_h, int Kh, int oh, const float* __restrict__ wts_w,
                const int* __restrict__ idx_w, int Kw, int ow, int TH, int TW, float* __restrict__ y) {
  extern __shared__ __align__(16) unsigned char dg_smem_raw[];
  const int tiles_x = (ow + TW - 1) / TW, tiles_y = (oh + TH - 1) / TH;
  const int f = blockIdx.x / (tiles_x * tiles_y), t = blockIdx.x - f * tiles_x * tiles_y;
  const int oy0 = t / tiles_x * TH, ox0 = t % tiles_x * TW;
  const int nr = min(TH, oh - oy0), nc = min(TW, ow - ox0);
  const int rows_cap = dg_span(TH, Kh, h), cols_cap = dg_span(TW, Kw, w);

  float* tw_h = reinterpret_cast<float*>(dg_smem_raw);
  int* ti_h = reinterpret_cast<int*>(tw_h + TH * Kh);
  float* tw_w = reinterpret_cast<float*>(ti_h + TH * Kh);
  int* ti_w = reinterpret_cast<int*>(tw_w + TW * Kw);
  float* unit = reinterpret_cast<float*>(ti_w + TW * Kw);
  uint8_t* src = reinterpret_cast<uint8_t*>(unit + 256);
  float* hp = reinterpret_cast<float*>(src + ((size_t)rows_cap * cols_cap * 3 + 15) / 16 * 16);   // [3][TH][cols]
  __shared__ int range[4];                                       // row lo, row hi, column lo, column hi

  if (threadIdx.x < 4) range[threadIdx.x] = (threadIdx.x & 1) ? -1 : 0x7fffffff;
  for (int v = threadIdx.x; v < 256; v += DG_THREADS) unit[v] = __double2float_rn(__ddiv_rn((double)v, 255.0));
  __syncthreads();
  int lo_r = 0x7fffffff, hi_r = -1, lo_c = 0x7fffffff, hi_c = -1;
  for (int i = threadIdx.x; i < nr * Kh; i += DG_THREADS) {
    const int v = __ldg(idx_h + (size_t)oy0 * Kh + i);
    tw_h[i] = __ldg(wts_h + (size_t)oy0 * Kh + i);
    lo_r = min(lo_r, v);
    hi_r = max(hi_r, v);
  }
  for (int i = threadIdx.x; i < nc * Kw; i += DG_THREADS) {
    const int v = __ldg(idx_w + (size_t)(ox0 + i / Kw) * Kw + i % Kw);
    tw_w[i] = __ldg(wts_w + (size_t)(ox0 + i / Kw) * Kw + i % Kw);
    lo_c = min(lo_c, v);
    hi_c = max(hi_c, v);
  }
  atomicMin(&range[0], lo_r);
  atomicMax(&range[1], hi_r);
  atomicMin(&range[2], lo_c);
  atomicMax(&range[3], hi_c);
  __syncthreads();
  const int r0 = range[0], c0 = range[2];
  const int rows = min(range[1] - r0 + 1, rows_cap), cols = min(range[3] - c0 + 1, cols_cap);
  // Indices relative to the footprint; the clamp only keeps a table that breaks dg_span's bound inside shared memory.
  for (int i = threadIdx.x; i < nr * Kh; i += DG_THREADS)
    ti_h[i] = min(__ldg(idx_h + (size_t)oy0 * Kh + i) - r0, rows - 1);
  for (int i = threadIdx.x; i < nc * Kw; i += DG_THREADS)
    ti_w[i] = min(__ldg(idx_w + (size_t)(ox0 + i / Kw) * Kw + i % Kw) - c0, cols - 1);

  // The footprint's rgb24 bytes: each source row's run of 3 cols bytes is contiguous.
  const uint8_t* frame = x + (size_t)f * h * w * 3;
  const int rb = cols * 3;
  for (int i = threadIdx.x; i < rows * rb; i += DG_THREADS) {
    const int r = i / rb, b = i - r * rb;
    src[i] = __ldg(frame + ((size_t)(r0 + r) * w + c0) * 3 + b);
  }
  __syncthreads();

  // H pass: out_1 of the tile's rows over the footprint's columns, items (row, column, channel), bytes consecutive.
  for (int i = threadIdx.x; i < nr * rb; i += DG_THREADS) {
    const int r = i / rb, b = i - r * rb;
    ExactSum acc;
    for (int k = 0; k < Kh; ++k) acc.add(tw_h[r * Kh + k], unit[src[ti_h[r * Kh + k] * rb + b]]);
    const int j = b / 3, c = b - j * 3;
    hp[((size_t)c * TH + r) * cols + j] = acc.value();
  }
  __syncthreads();

  // W pass: items (channel, row, column), columns fastest for coalesced stores.
  const size_t plane = (size_t)oh * ow;
  float* dst = y + (size_t)f * 3 * plane;
  for (int i = threadIdx.x; i < 3 * nr * nc; i += DG_THREADS) {
    const int cr = i / nc, ox = i - cr * nc, c = cr / nr, r = cr - c * nr;
    const float* row = hp + ((size_t)c * TH + r) * cols;
    ExactSum acc;
    for (int k = 0; k < Kw; ++k) acc.add(tw_w[ox * Kw + k], row[ti_w[ox * Kw + k]]);
    dst[c * plane + (size_t)(oy0 + r) * ow + ox0 + ox] = acc.value();
  }
}

}  // namespace pgt

using namespace pgt;

extern "C" int pgt_imresize_u8hwc_to_f32nchw(const void* x_u8, int F, int h, int w, const float* wts_h,
                                             const int32_t* idx_h, int Kh, int oh, const float* wts_w,
                                             const int32_t* idx_w, int Kw, int ow, float* y, void* stream) {
  PGT_CHECK_ARG(x_u8 && y && wts_h && idx_h && wts_w && idx_w && F > 0 && h > 0 && w > 0);
  PGT_CHECK_ARG(Kh > 0 && Kw > 0 && Kh <= 256 && Kw <= 256 && oh > 0 && ow > 0 && oh <= h && ow <= w);
  int TH = 16, TW = 32;
  while (dg_smem(TH, TW, Kh, Kw, h, w) > (size_t)DG_SMEM_MAX && (TH > 1 || TW > 1)) {
    if (TW >= TH) TW /= 2; else TH /= 2;
  }
  const size_t smem = dg_smem(TH, TW, Kh, Kw, h, w);
  PGT_CHECK_ARG(smem <= (size_t)DG_SMEM_MAX);
  const long long tiles = (long long)((oh + TH - 1) / TH) * ((ow + TW - 1) / TW);
  PGT_CHECK_ARG((long long)F * tiles <= 0x7fffffffLL);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  static PerDeviceOnce once;                               // above the default 48 KB of dynamic shared memory
  PGT_CUDA_OK(once.run([] {
    return cudaFuncSetAttribute(imresize_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, DG_SMEM_MAX);
  }));
  ProfScope ps(PGT_PROF_MOVE, 3.0 * F * (double)h * w + 12.0 * F * (double)oh * ow, st,
               "pgt_imresize_u8hwc_to_f32nchw");
  imresize_kernel<<<(unsigned)(F * tiles), DG_THREADS, smem, st>>>(static_cast<const uint8_t*>(x_u8), h, w, wts_h,
                                                                    idx_h, Kh, oh, wts_w, idx_w, Kw, ow, TH, TW, y);
  PGT_LAUNCH_OK();
  return PGT_OK;
}
