// Kernels specific to the face-parsing branch (BiSeNet / ResNet18, archs/pgtformer_arch.py:34-397 in the
// reference): 3x3 stride-2 max-pool, global average pool, per-(frame,channel)
// attention re-weighting, and the bilinear(align_corners) assembly of the three 19-class heads into the
// 57(+7 pad)-channel conditioning map.  Every convolution of the branch (the 7x7 stem included) runs on the wgmma
// kernels with BatchNorm folded into weights / bias.
#include <float.h>

#include "common.cuh"

namespace pgt {

__device__ __forceinline__ void ld8(const __nv_bfloat16* p, float (&v)[8]) {
  const uint4 u = __ldg(reinterpret_cast<const uint4*>(p));
  float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
}
__device__ __forceinline__ void st8(__nv_bfloat16* p, const float (&v)[8]) {
  uint4 u;
  u.x = pack_bf16x2(v[0], v[1]); u.y = pack_bf16x2(v[2], v[3]);
  u.z = pack_bf16x2(v[4], v[5]); u.w = pack_bf16x2(v[6], v[7]);
  *reinterpret_cast<uint4*>(p) = u;
}

// ------------------------------------------------------------------------------ 3x3 s2 p1 max-pool
__global__ void maxpool3x3s2_kernel(const __nv_bfloat16* __restrict__ x, int ldx, int F, int H, int W, int C,
                                    __nv_bfloat16* __restrict__ y, int ldy) {
  const int Ho = H >> 1, Wo = W >> 1, vc = C >> 3;
  const size_t total = (size_t)F * Ho * Wo * vc;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int v = (int)(i % vc);
    size_t pix = i / vc;
    const int ox = (int)(pix % Wo); pix /= Wo;
    const int oy = (int)(pix % Ho);
    const int f = (int)(pix / Ho);
    float m[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) m[j] = -FLT_MAX;
#pragma unroll
    for (int dy = 0; dy < 3; ++dy) {
      const int iy = 2 * oy - 1 + dy;
      if (iy < 0 || iy >= H) continue;
#pragma unroll
      for (int dx = 0; dx < 3; ++dx) {
        const int ix = 2 * ox - 1 + dx;
        if (ix < 0 || ix >= W) continue;
        float t[8];
        ld8(x + (((size_t)f * H + iy) * W + ix) * ldx + v * 8, t);
#pragma unroll
        for (int j = 0; j < 8; ++j) m[j] = fmaxf(m[j], t[j]);
      }
    }
    st8(y + (((size_t)f * Ho + oy) * Wo + ox) * ldy + v * 8, m);
  }
}

// ------------------------------------------------------------------------------ global average pool -> [F, C] bf16
__global__ void __launch_bounds__(256)
global_avgpool_kernel(const __nv_bfloat16* __restrict__ x, int ldx, int HW, int C, __nv_bfloat16* __restrict__ y, int ldy) {
  __shared__ float red[32][64];
  const int f = blockIdx.y, cbase = blockIdx.x * 64;
  const int vcol = threadIdx.x & 7, prow = threadIdx.x >> 3;
  const int c0 = cbase + vcol * 8;
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  if (c0 < C) {
    for (int p = prow; p < HW; p += 32) {
      float v[8];
      ld8(x + ((size_t)f * HW + p) * ldx + c0, v);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += v[j];
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) red[prow][vcol * 8 + j] = acc[j];
  __syncthreads();
  if (threadIdx.x < 64 && cbase + threadIdx.x < C) {
    float s = 0.f;
    for (int r = 0; r < 32; ++r) s += red[r][threadIdx.x];
    y[(size_t)f * ldy + cbase + threadIdx.x] = __float2bfloat16_rn(s / (float)HW);
  }
}

// ------------------------------------------------------------------------------ y = x * (scale[f,c] (+1)) + addv[f,c] + addm
__global__ void channel_affine_kernel(const __nv_bfloat16* __restrict__ x, int ldx, int F, int HW, int C,
                                      const __nv_bfloat16* __restrict__ scale, int lds, int plus_one,
                                      const __nv_bfloat16* __restrict__ addv, int ldv,
                                      const __nv_bfloat16* __restrict__ addm, int ldm, __nv_bfloat16* __restrict__ y, int ldy) {
  const int vc = C >> 3;
  const size_t total = (size_t)F * HW * vc;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int v = (int)(i % vc);
    const size_t pix = i / vc;
    const int f = (int)(pix / HW);
    float a[8], s[8];
    ld8(x + pix * ldx + v * 8, a);
    ld8(scale + (size_t)f * lds + v * 8, s);
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] *= (plus_one ? s[j] + 1.f : s[j]);
    if (addv != nullptr) {
      float t[8];
      ld8(addv + (size_t)f * ldv + v * 8, t);
#pragma unroll
      for (int j = 0; j < 8; ++j) a[j] += t[j];
    }
    if (addm != nullptr) {
      float t[8];
      ld8(addm + pix * ldm + v * 8, t);
#pragma unroll
      for (int j = 0; j < 8; ++j) a[j] += t[j];
    }
    st8(y + pix * ldy + v * 8, a);
  }
}

// ------------------------------------------------------------------------------ heads -> conditioning map
// cond[f, y, x, 0:19]  = bilinear(align_corners) of o0 (h8 x w8) ; [19:38] = bilinear of o1 ; [38:57] = o2 ; [57:64] = 0
__global__ void assemble_cond_kernel(const __nv_bfloat16* __restrict__ o0, int ld0, const __nv_bfloat16* __restrict__ o1,
                                     int ld1, const __nv_bfloat16* __restrict__ o2, int ld2, int F, int h8, int w8, int h16,
                                     int w16, int ncls, __nv_bfloat16* __restrict__ cond, int ldc) {
  const size_t total = (size_t)F * h16 * w16 * 64;
  const float sy = h16 > 1 ? (float)(h8 - 1) / (float)(h16 - 1) : 0.f;
  const float sx = w16 > 1 ? (float)(w8 - 1) / (float)(w16 - 1) : 0.f;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i & 63);
    size_t pix = i >> 6;
    const int x = (int)(pix % w16); pix /= w16;
    const int y = (int)(pix % h16);
    const int f = (int)(pix / h16);
    float v = 0.f;
    if (c < 2 * ncls) {
      const __nv_bfloat16* src = c < ncls ? o0 : o1;
      const int ld = c < ncls ? ld0 : ld1;
      const int ch = c < ncls ? c : c - ncls;
      const float fy = y * sy, fx = x * sx;
      const int y0 = (int)fy, x0 = (int)fx;
      const int y1 = min(y0 + 1, h8 - 1), x1 = min(x0 + 1, w8 - 1);
      const float ly = fy - y0, lx = fx - x0;
      auto at = [&](int yy, int xx) { return __bfloat162float(src[(((size_t)f * h8 + yy) * w8 + xx) * ld + ch]); };
      v = (1.f - ly) * ((1.f - lx) * at(y0, x0) + lx * at(y0, x1)) + ly * ((1.f - lx) * at(y1, x0) + lx * at(y1, x1));
    } else if (c < 3 * ncls) {
      v = __bfloat162float(o2[(((size_t)f * h16 + y) * w16 + x) * ld2 + (c - 2 * ncls)]);
    }
    cond[(((size_t)f * h16 + y) * w16 + x) * ldc + c] = __float2bfloat16_rn(v);
  }
}

}  // namespace pgt

using namespace pgt;

static int grid_for(size_t total, int threads) {
  size_t b = (total + threads - 1) / threads;
  const size_t cap = (size_t)num_sms() * 32;
  return (int)(b < cap ? (b ? b : 1) : cap);
}

extern "C" int pgt_maxpool3x3s2(const void* x, int ldx, int F, int H, int W, int C, void* y, int ldy, void* stream) {
  PGT_CHECK_ARG(x && y && F > 0 && (H % 2) == 0 && (W % 2) == 0 && C % 8 == 0 && ldx % 8 == 0 && ldy % 8 == 0);
  const size_t total = (size_t)F * (H / 2) * (W / 2) * (C / 8);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ProfScope ps(PGT_PROF_MOVE, 2.5 * F * (double)H * W * C, st, "maxpool");
  maxpool3x3s2_kernel<<<grid_for(total, 256), 256, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(x), ldx, F, H, W, C,
                                                           reinterpret_cast<__nv_bfloat16*>(y), ldy);
  PGT_LAUNCH_OK();
  return PGT_OK;
}

extern "C" int pgt_global_avgpool(const void* x, int ldx, int F, int HW, int C, void* y, int ldy, void* stream) {
  PGT_CHECK_ARG(x && y && F > 0 && HW > 0 && C % 8 == 0 && ldx % 8 == 0 && ldy >= C);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ProfScope ps(PGT_PROF_MOVE, 2.0 * F * (double)HW * C, st, "avgpool");
  global_avgpool_kernel<<<dim3(ceil_div(C, 64), F), 256, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(x), ldx, HW, C,
                                                                 reinterpret_cast<__nv_bfloat16*>(y), ldy);
  PGT_LAUNCH_OK();
  return PGT_OK;
}

extern "C" int pgt_channel_affine(const void* x, int ldx, int F, int HW, int C, const void* scale, int lds, int plus_one,
                                  const void* addv, int ldv, const void* addm, int ldm, void* y, int ldy, void* stream) {
  PGT_CHECK_ARG(x && y && scale && F > 0 && HW > 0 && C % 8 == 0 && ldx % 8 == 0 && ldy % 8 == 0 && lds % 8 == 0);
  PGT_CHECK_ARG((addv == nullptr || ldv % 8 == 0) && (addm == nullptr || ldm % 8 == 0));
  const size_t total = (size_t)F * HW * (C / 8);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ProfScope ps(PGT_PROF_MOVE, (addm ? 6.0 : 4.0) * F * (double)HW * C, st, "channel_affine");
  channel_affine_kernel<<<grid_for(total, 256), 256, 0, st>>>(
      reinterpret_cast<const __nv_bfloat16*>(x), ldx, F, HW, C, reinterpret_cast<const __nv_bfloat16*>(scale), lds, plus_one,
      reinterpret_cast<const __nv_bfloat16*>(addv), ldv, reinterpret_cast<const __nv_bfloat16*>(addm), ldm,
      reinterpret_cast<__nv_bfloat16*>(y), ldy);
  PGT_LAUNCH_OK();
  return PGT_OK;
}

extern "C" int pgt_assemble_cond(const void* o0, int ld0, const void* o1, int ld1, const void* o2, int ld2, int F, int h8,
                                 int w8, int h16, int w16, int ncls, void* cond, int ldc, void* stream) {
  PGT_CHECK_ARG(o0 && o1 && o2 && cond && F > 0 && h8 > 0 && w8 > 0 && h16 > 0 && w16 > 0 && ncls > 0 && 3 * ncls <= 64 &&
                ldc >= 64);
  const size_t total = (size_t)F * h16 * w16 * 64;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ProfScope ps(PGT_PROF_MOVE, 4.0 * (double)total, st, "assemble_cond");
  assemble_cond_kernel<<<grid_for(total, 256), 256, 0, st>>>(
      reinterpret_cast<const __nv_bfloat16*>(o0), ld0, reinterpret_cast<const __nv_bfloat16*>(o1), ld1,
      reinterpret_cast<const __nv_bfloat16*>(o2), ld2, F, h8, w8, h16, w16, ncls, reinterpret_cast<__nv_bfloat16*>(cond), ldc);
  PGT_LAUNCH_OK();
  return PGT_OK;
}
