// Layout conversion and small data-movement kernels (HBM-bound, 128-bit vectorised), and the streaming video
// front / back end.
#include <algorithm>

#include "common.cuh"
#include "tmap.cuh"

namespace pgt {

__global__ void copy2d_kernel(const __nv_bfloat16* __restrict__ x, int ldx, size_t T, int C,
                              __nv_bfloat16* __restrict__ y, int ldy) {
  const int vc = C >> 3;
  const size_t total = T * vc;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (; i + 3 * stride < total; i += 4 * stride) {       // four independent 16-byte copies in flight
    uint4 u[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const size_t j = i + k * stride;
      u[k] = __ldg(reinterpret_cast<const uint4*>(x + (j / vc) * ldx) + (j % vc));
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const size_t j = i + k * stride;
      reinterpret_cast<uint4*>(y + (j / vc) * ldy)[j % vc] = u[k];
    }
  }
  for (; i < total; i += stride)
    reinterpret_cast<uint4*>(y + (i / vc) * ldy)[i % vc] = __ldg(reinterpret_cast<const uint4*>(x + (i / vc) * ldx) + (i % vc));
}

// fp32 NCHW -> bf16 NHWC through a 32x32 shared-memory transpose (coalesced on both sides).
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ x, int C, int HW, const float* __restrict__ mean,
                                    const float* __restrict__ stdv, __nv_bfloat16* __restrict__ y, int ldy) {
  __shared__ float tile[32][33];
  const int f = blockIdx.z;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int c = c0 + j, p = p0 + threadIdx.x;
    float v = 0.f;
    if (c < C && p < HW) {
      v = x[((size_t)f * C + c) * HW + p];
      if (mean != nullptr) v = (v - mean[c]) / stdv[c];
    }
    tile[j][threadIdx.x] = v;
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int p = p0 + j, c = c0 + threadIdx.x;
    if (p < HW && c < ldy && c0 + 32 <= ((C + 31) / 32) * 32) {
      if (c < C) y[((size_t)f * HW + p) * ldy + c] = __float2bfloat16_rn(tile[threadIdx.x][j]);
    }
  }
}

__global__ void nhwc_to_f32_kernel(const __nv_bfloat16* __restrict__ x, int ldx, int HW, int C, float* __restrict__ y,
                                   int to_nchw) {
  __shared__ float tile[32][33];
  const int f = blockIdx.z;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int p = p0 + j, c = c0 + threadIdx.x;
    tile[j][threadIdx.x] = (p < HW && c < C) ? __bfloat162float(x[((size_t)f * HW + p) * ldx + c]) : 0.f;
  }
  __syncthreads();
  if (to_nchw) {
    for (int j = threadIdx.y; j < 32; j += blockDim.y) {
      const int c = c0 + j, p = p0 + threadIdx.x;
      if (c < C && p < HW) y[((size_t)f * C + c) * HW + p] = tile[threadIdx.x][j];
    }
  } else {
    for (int j = threadIdx.y; j < 32; j += blockDim.y) {
      const int p = p0 + j, c = c0 + threadIdx.x;
      if (c < C && p < HW) y[((size_t)f * HW + p) * C + c] = tile[j][threadIdx.x];
    }
  }
}

}  // namespace pgt

using namespace pgt;

static int ew_grid(size_t total, int threads) {
  size_t b = (total + threads - 1) / threads;
  const size_t cap = (size_t)num_sms() * 32;
  return (int)(b < cap ? (b ? b : 1) : cap);
}

extern "C" int pgt_copy2d(const void* x, int ldx, int T, int C, void* y, int ldy, void* stream) {
  PGT_CHECK_ARG(x && y && T > 0 && C % 8 == 0 && ldx % 8 == 0 && ldy % 8 == 0);
  ProfScope ps(PGT_PROF_MOVE, 2.0 * (double)T * C * 2, static_cast<cudaStream_t>(stream), "pgt_copy2d");
  const size_t total = (size_t)T * (C / 8);
  copy2d_kernel<<<ew_grid(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(x), ldx, (size_t)T, C, reinterpret_cast<__nv_bfloat16*>(y), ldy);
  PGT_LAUNCH_OK();
  return PGT_OK;
}

extern "C" int pgt_nchw_f32_to_nhwc_bf16(const float* x, int F, int C, int HW, const float* mean, const float* stdv,
                                         void* y, int ldy, void* stream) {
  PGT_CHECK_ARG(x && y && F > 0 && C > 0 && HW > 0 && ldy >= C && (mean == nullptr) == (stdv == nullptr));
  ProfScope ps(PGT_PROF_MOVE, 6.0 * F * (double)C * HW, static_cast<cudaStream_t>(stream), "pgt_nchw_f32_to_nhwc_bf16");
  dim3 grid(ceil_div(HW, 32), ceil_div(C, 32), F);
  nchw_to_nhwc_kernel<<<grid, dim3(32, 8), 0, static_cast<cudaStream_t>(stream)>>>(
      x, C, HW, mean, stdv, reinterpret_cast<__nv_bfloat16*>(y), ldy);
  PGT_LAUNCH_OK();
  return PGT_OK;
}

extern "C" int pgt_nhwc_bf16_to_f32(const void* x, int ldx, int F, int HW, int C, float* y, int to_nchw, void* stream) {
  PGT_CHECK_ARG(x && y && F > 0 && C > 0 && HW > 0 && ldx >= C);
  ProfScope ps(PGT_PROF_MOVE, 6.0 * F * (double)C * HW, static_cast<cudaStream_t>(stream), "pgt_nhwc_bf16_to_f32");
  dim3 grid(ceil_div(HW, 32), ceil_div(C, 32), F);
  nhwc_to_f32_kernel<<<grid, dim3(32, 8), 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(x), ldx, HW, C, y, to_nchw);
  PGT_LAUNCH_OK();
  return PGT_OK;
}

// ---- temporal regroup used by the SFT fusion block's cross-frame 1x1 mixers
// dir 0: x [b,3,P,C] -> y [b,P,3*C] (channel = frame*C + c);   dir 1: the inverse.
namespace pgt {
__global__ void regroup_frames_kernel(const __nv_bfloat16* __restrict__ x, int ldx, int b, int P, int C,
                                      __nv_bfloat16* __restrict__ y, int ldy, int dir) {
  const int vc = C >> 3;
  const size_t total = (size_t)b * 3 * P * vc;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int v = (int)(i % vc);
    size_t r = i / vc;
    const int p = (int)(r % P); r /= P;
    const int fr = (int)(r % 3);
    const int clip = (int)(r / 3);
    const size_t frame_row = ((size_t)clip * 3 + fr) * P + p;          // [b,3,P] row
    const size_t clip_row = (size_t)clip * P + p;                      // [b,P] row
    if (dir == 0)
      reinterpret_cast<uint4*>(y + clip_row * ldy + fr * C)[v] = __ldg(reinterpret_cast<const uint4*>(x + frame_row * ldx) + v);
    else
      reinterpret_cast<uint4*>(y + frame_row * ldy)[v] = __ldg(reinterpret_cast<const uint4*>(x + clip_row * ldx + fr * C) + v);
  }
}
}  // namespace pgt

extern "C" int pgt_regroup_frames(const void* x, int ldx, int clips, int P, int C, void* y, int ldy, int dir,
                                  void* stream) {
  PGT_CHECK_ARG(x && y && clips > 0 && P > 0 && C % 8 == 0 && ldx % 8 == 0 && ldy % 8 == 0 && (dir == 0 || dir == 1));
  ProfScope ps(PGT_PROF_MOVE, 4.0 * clips * 3.0 * P * C, static_cast<cudaStream_t>(stream), "pgt_regroup_frames");
  const size_t total = (size_t)clips * 3 * P * (C / 8);
  regroup_frames_kernel<<<ew_grid(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(x), ldx, clips, P, C, reinterpret_cast<__nv_bfloat16*>(y), ldy, dir);
  PGT_LAUNCH_OK();
  return PGT_OK;
}


// ---------------------------------------------------------------- streaming video front / back end
// The reference's loop (inference.py:6-19,37-76) turns rgb24 frames into float tensors with numpy
// (`np.array(rgb / 255.0, np.float32)`: a double division rounded to fp32), runs the model on the window
// (f[i-1], f[i], f[i+1]) and writes `clamp(out[0][1], 0, 1) * 255` truncated to uint8.  These kernels are those two
// conversions, and the frame gather that lets per-frame work (BiSeNet, the attention-free encoder levels) be computed
// once per distinct frame and handed to every window that contains the frame.
namespace pgt {
__constant__ float c_u8_to_unit[256];             // (float)(v / 255.0) evaluated in double on the host

__global__ void u8hwc_to_f32nchw_kernel(const uint8_t* __restrict__ x, size_t HW, size_t total, float* __restrict__ y) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t f = i / HW, p = i - f * HW;
    const uint8_t* s = x + (f * HW + p) * 3;
    float* d = y + f * 3 * HW + p;
    d[0] = c_u8_to_unit[s[0]];
    d[HW] = c_u8_to_unit[s[1]];
    d[2 * HW] = c_u8_to_unit[s[2]];
  }
}

__global__ void f32nchw_to_u8hwc_kernel(const float* __restrict__ x, size_t HW, int first, int step, size_t total,
                                        uint8_t* __restrict__ y) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t j = i / HW, p = i - j * HW;
    const float* s = x + ((size_t)first + j * step) * 3 * HW + p;
    uint8_t* d = y + (j * HW + p) * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float v = fminf(fmaxf(s[c * HW], 0.f), 1.f) * 255.0f;     // torch.clamp, then the fp32 product numpy forms
      d[c] = (uint8_t)v;                                             // astype(uint8) of a value in [0, 255]: truncation
    }
  }
}

__global__ void gather_frames_kernel(const uint4* __restrict__ x, size_t vec_per_frame, const int* __restrict__ idx,
                                     uint4* __restrict__ y) {
  const uint4* s = x + (size_t)idx[blockIdx.y] * vec_per_frame;
  uint4* d = y + (size_t)blockIdx.y * vec_per_frame;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < vec_per_frame; i += (size_t)gridDim.x * blockDim.x)
    d[i] = __ldg(s + i);
}

__global__ void scatter_frames_kernel(const uint4* __restrict__ x, size_t vec_per_frame, const int* __restrict__ idx,
                                      uint4* __restrict__ y) {
  const uint4* s = x + (size_t)blockIdx.y * vec_per_frame;
  uint4* d = y + (size_t)idx[blockIdx.y] * vec_per_frame;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < vec_per_frame; i += (size_t)gridDim.x * blockDim.x)
    d[i] = __ldg(s + i);
}

// The low-resolution input of the reference's test set (data/vfhq_full_dataset.py:1046-1051): rgb24 frames of any
// size, (float)(v / 255.0), then F.interpolate(mode='bilinear', align_corners=True) to the model's H x W.  One output
// axis position o maps to source rows i0, i1 with weights l0, l1 exactly as torch's CPU kernel computes them, every
// step in fp32: scale = (in - 1) / (out - 1) (0 for out = 1), src = scale * o, i0 = min(floor(src), in - 1),
// i1 = i0 + (i0 < in - 1), l1 = clamp(src - i0, 0, 1), l0 = 1 - l1.
struct LerpAxis {
  int i0, i1;
  float l0, l1;
};

__device__ __forceinline__ LerpAxis lerp_axis(int in, int out, int o) {
  const float scale = out > 1 ? __fdiv_rn((float)(in - 1), (float)(out - 1)) : 0.f;
  const float src = __fmul_rn(scale, (float)o);
  LerpAxis a;
  a.i0 = min((int)floorf(src), in - 1);
  a.i1 = a.i0 + (a.i0 < in - 1 ? 1 : 0);
  a.l1 = fminf(fmaxf(__fsub_rn(src, (float)a.i0), 0.f), 1.f);
  a.l0 = __fsub_rn(1.f, a.l1);
  return a;
}

// The source of a resize: frame f's size and (c, y, x) sample as the fp32 value the interpolation reads.
//   U8Frames: rgb24 frames, (float)(v / 255.0) through the CTA's table `unit`; every frame h x w packed one after
//     another, or each frame's (h, w, byte offset) from a device int32 table.
//   F32Planes: fp32 frames [F, 3, h, w] (the output of pgt_imresize_u8hwc_to_f32nchw); `unit` is not read.
struct U8Frames {
  static constexpr bool kUnit = true;
  const uint8_t* x;
  int h, w;
  const int* sizes;
  struct Frame {
    const uint8_t* p;
    int h, w;
  };
  __device__ __forceinline__ Frame frame(int f) const {
    if (sizes == nullptr) return {x + (size_t)f * h * w * 3, h, w};
    return {x + (size_t)(unsigned)__ldg(sizes + 3 * f + 2), __ldg(sizes + 3 * f), __ldg(sizes + 3 * f + 1)};
  }
  __device__ __forceinline__ float at(const Frame& fr, const float* unit, int c, int y, int xx) const {
    return unit[fr.p[((size_t)y * fr.w + xx) * 3 + c]];
  }
};

struct F32Planes {
  static constexpr bool kUnit = false;
  const float* x;
  int h, w;
  struct Frame {
    const float* p;
    int h, w;
  };
  __device__ __forceinline__ Frame frame(int f) const { return {x + (size_t)f * 3 * h * w, h, w}; }
  __device__ __forceinline__ float at(const Frame& fr, const float*, int c, int y, int xx) const {
    return __ldg(fr.p + ((size_t)c * fr.h + y) * fr.w + xx);
  }
};

// Each thread writes four consecutive pixels of one output row (W % 4 == 0), all three planes, as float4 stores.
// The combination is the one torch's AVX2 / AVX512 kernel evaluates, fma(h0, fma(w0, a, w1 b), h1 fma(w0, c, w1 d)),
// spelled with explicit intrinsics so that no contraction choice of the compiler changes a bit.
template <class Src>
__global__ void resize_kernel(Src src, int H, int W, size_t total, float* __restrict__ y) {
  __shared__ float unit[Src::kUnit ? 256 : 1];
  if (Src::kUnit) {
    for (int v = threadIdx.x; v < 256; v += blockDim.x) unit[v] = __double2float_rn(__ddiv_rn((double)v, 255.0));
    __syncthreads();
  }
  const int qw = W >> 2;
  const size_t HW = (size_t)H * W;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t row = i / qw;
    const int ox = (int)(i - row * qw) << 2;
    const int f = (int)(row / H), oy = (int)(row - (size_t)f * H);
    const typename Src::Frame fr = src.frame(f);
    const LerpAxis ay = lerp_axis(fr.h, H, oy);
    float o[3][4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const LerpAxis ax = lerp_axis(fr.w, W, ox + k);
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float a = src.at(fr, unit, c, ay.i0, ax.i0), b = src.at(fr, unit, c, ay.i0, ax.i1);
        const float cc = src.at(fr, unit, c, ay.i1, ax.i0), d = src.at(fr, unit, c, ay.i1, ax.i1);
        const float top = __fmaf_rn(ax.l0, a, __fmul_rn(ax.l1, b));
        const float bot = __fmaf_rn(ax.l0, cc, __fmul_rn(ax.l1, d));
        o[c][k] = __fmaf_rn(ay.l0, top, __fmul_rn(ay.l1, bot));
      }
    }
    float* dst = y + (size_t)f * 3 * HW + (size_t)oy * W + ox;
#pragma unroll
    for (int c = 0; c < 3; ++c)
      *reinterpret_cast<float4*>(dst + c * HW) = make_float4(o[c][0], o[c][1], o[c][2], o[c][3]);
  }
}
}  // namespace pgt

extern "C" int pgt_u8hwc_to_f32nchw(const void* x_u8, int F, int H, int W, float* y, void* stream) {
  PGT_CHECK_ARG(x_u8 && y && F > 0 && H > 0 && W > 0);
  static pgt::PerDeviceOnce once;               // __constant__ memory is per device
  PGT_CUDA_OK(once.run([] {
    float t[256];
    for (int v = 0; v < 256; ++v) t[v] = (float)((double)v / 255.0);
    return cudaMemcpyToSymbol(pgt::c_u8_to_unit, t, sizeof(t));
  }));
  const size_t HW = (size_t)H * W, total = (size_t)F * HW;
  ProfScope ps(PGT_PROF_MOVE, 15.0 * (double)total, static_cast<cudaStream_t>(stream), "pgt_u8hwc_to_f32nchw");
  pgt::u8hwc_to_f32nchw_kernel<<<ew_grid(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const uint8_t*>(x_u8), HW, total, y);
  PGT_LAUNCH_OK();
  return PGT_OK;
}

extern "C" int pgt_u8hwc_resize_to_f32nchw(const void* x_u8, int F, int h, int w, const int32_t* sizes_dev, int H,
                                           int W, float* y, void* stream) {
  PGT_CHECK_ARG(x_u8 && y && F > 0 && h > 0 && w > 0 && H > 0 && W > 0 && H % 64 == 0 && W % 64 == 0);
  PGT_CHECK_ARG((reinterpret_cast<uintptr_t>(y) & 15) == 0);
  const size_t total = (size_t)F * H * (W / 4);
  ProfScope ps(PGT_PROF_MOVE, 12.0 * F * (double)H * W + 3.0 * F * (double)h * w, static_cast<cudaStream_t>(stream),
               "pgt_u8hwc_resize_to_f32nchw");
  pgt::resize_kernel<<<ew_grid(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      pgt::U8Frames{static_cast<const uint8_t*>(x_u8), h, w, sizes_dev}, H, W, total, y);
  PGT_LAUNCH_OK();
  return PGT_OK;
}

extern "C" int pgt_f32nchw_resize_to_f32nchw(const float* x, int F, int h, int w, int H, int W, float* y,
                                             void* stream) {
  PGT_CHECK_ARG(x && y && F > 0 && h > 0 && w > 0 && H > 0 && W > 0 && H % 64 == 0 && W % 64 == 0);
  PGT_CHECK_ARG((reinterpret_cast<uintptr_t>(y) & 15) == 0);
  const size_t total = (size_t)F * H * (W / 4);
  ProfScope ps(PGT_PROF_MOVE, 12.0 * F * (double)H * W + 12.0 * F * (double)h * w, static_cast<cudaStream_t>(stream),
               "pgt_f32nchw_resize_to_f32nchw");
  pgt::resize_kernel<<<ew_grid(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      pgt::F32Planes{x, h, w}, H, W, total, y);
  PGT_LAUNCH_OK();
  return PGT_OK;
}

extern "C" int pgt_f32nchw_to_u8hwc(const float* x, int first, int step, int n, int H, int W, void* y_u8, void* stream) {
  PGT_CHECK_ARG(x && y_u8 && n > 0 && H > 0 && W > 0 && first >= 0 && step >= 1);
  const size_t HW = (size_t)H * W, total = (size_t)n * HW;
  ProfScope ps(PGT_PROF_MOVE, 15.0 * (double)total, static_cast<cudaStream_t>(stream), "pgt_f32nchw_to_u8hwc");
  pgt::f32nchw_to_u8hwc_kernel<<<ew_grid(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x, HW, first, step, total, static_cast<uint8_t*>(y_u8));
  PGT_LAUNCH_OK();
  return PGT_OK;
}

extern "C" int pgt_gather_frames(const void* x, long long frame_bytes, const int* idx_dev, int n, void* y, void* stream) {
  PGT_CHECK_ARG(x && y && idx_dev && n > 0 && frame_bytes > 0 && frame_bytes % 16 == 0);
  PGT_CHECK_ARG((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(y) & 15) == 0);
  const size_t vec = (size_t)frame_bytes / 16;
  ProfScope ps(PGT_PROF_MOVE, 2.0 * (double)n * frame_bytes, static_cast<cudaStream_t>(stream), "pgt_gather_frames");
  unsigned bx = (unsigned)std::min<size_t>((vec + 255) / 256, 1024);
  pgt::gather_frames_kernel<<<dim3(bx, n), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const uint4*>(x), vec, idx_dev, static_cast<uint4*>(y));
  PGT_LAUNCH_OK();
  return PGT_OK;
}

extern "C" int pgt_scatter_frames(const void* x, long long frame_bytes, const int* idx_dev, int n, void* y, void* stream) {
  PGT_CHECK_ARG(x && y && idx_dev && n > 0 && frame_bytes > 0 && frame_bytes % 16 == 0);
  PGT_CHECK_ARG((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(y) & 15) == 0);
  const size_t vec = (size_t)frame_bytes / 16;
  ProfScope ps(PGT_PROF_MOVE, 2.0 * (double)n * frame_bytes, static_cast<cudaStream_t>(stream), "pgt_scatter_frames");
  unsigned bx = (unsigned)std::min<size_t>((vec + 255) / 256, 1024);
  pgt::scatter_frames_kernel<<<dim3(bx, n), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const uint4*>(x), vec, idx_dev, static_cast<uint4*>(y));
  PGT_LAUNCH_OK();
  return PGT_OK;
}
