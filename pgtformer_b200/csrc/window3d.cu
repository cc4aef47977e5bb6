// Generic 3-D shifted-window attention core for the Video-Swin `BasicLayer` of the reference's TDRQVAE
// (`modules/swin.py:136-166` WindowAttention3D.forward, `:214-250` pad / roll / partition / reverse / crop,
// `:309-323` compute_mask): any window (wd, wh, ww) with N = wd*wh*ww <= 128 tokens, any shift, feature maps that are
// NOT multiples of the window (zero padding after the norm, exactly as the reference pads), bias through the
// `relative_position_index[:N, :N]` slice (expanded on the host).
//
// This is the widening row SURVEY 8(f) #4, not the hot path: TDRQVAE runs two such layers on the 32x32 latent grid
// only.  One CTA per (window, head); q / k / v rows of the head are gathered into shared memory (padded tokens take the
// projection of a zero row, i.e. the qkv bias or zero), a warp owns 16 query rows: S = q k^T and O = P v on
// mma.sync.m16n8k16 with fp32 softmax in registers.  The wgmma kernel of window_attn_tc.cu is specialised to the
// 3x4x4 windows of the PGTFormer path (N = 48 fills TMA boxes and wgmma tiles exactly); N = 75 with padding does not.
#include "common.cuh"
#include "tmap.cuh"

namespace pgt {

__device__ __forceinline__ void w3_mma_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void w3_ldmatrix_x2_trans(uint32_t& r0, uint32_t& r1, const void* smem_row_ptr) {
  const uint32_t a = static_cast<uint32_t>(__cvta_generic_to_shared(smem_row_ptr));
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0,%1}, [%2];" : "=r"(r0), "=r"(r1) : "r"(a));
}

struct Win3dParams {
  const __nv_bfloat16* qkv;      // [B*D*H*W, ldqkv]: q | k | v, each C wide
  int ldqkv;
  const __nv_bfloat16* pad_qkv;  // [3C] projection of a zero token (qkv bias) or null (= zeros)
  const float* bias;             // [heads, N, N] expanded relative-position bias
  __nv_bfloat16* out;            // [B*D*H*W, ldo]
  int ldo;
  int B, D, H, W, C, heads;
  int wd, wh, ww, sd, sh, sw;    // effective window / shift (after get_window_size)
  int Dp, Hp, Wp, nd, nh, nw;    // padded extents, windows per dimension
  int N, NP;                     // tokens per window, rounded up to 16
};

constexpr int W3_MAXNP = 128;

template <int HD>
__global__ void __launch_bounds__(256)
window3d_attn_kernel(const Win3dParams p) {
  constexpr int LDS = HD + 8;                                   // padded smem row (bf16)
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __nv_bfloat16* qs = reinterpret_cast<__nv_bfloat16*>(smem_raw);          // [NP][LDS]
  __nv_bfloat16* ks = qs + W3_MAXNP * LDS;
  __nv_bfloat16* vs = ks + W3_MAXNP * LDS;
  __shared__ int tok[W3_MAXNP];
  __shared__ int lab[W3_MAXNP];
  const int win = blockIdx.x, h = blockIdx.y;
  const int per_b = p.nd * p.nh * p.nw;
  const int b = win / per_b;
  int r = win - b * per_b;
  const int wz = r / (p.nh * p.nw);
  r -= wz * p.nh * p.nw;
  const int wy = r / p.nw, wx = r - wy * p.nw;
  const bool shifted = (p.sd | p.sh | p.sw) != 0;
  if (threadIdx.x < p.NP) {
    const int i = threadIdx.x;
    int t = -1, l = 0;
    if (i < p.N) {
      const int id = i / (p.wh * p.ww), ih = (i / p.ww) % p.wh, iw = i % p.ww;
      const int pd = wz * p.wd + id, ph = wy * p.wh + ih, pw = wx * p.ww + iw;     // position in the shifted, padded frame
      const int d = (pd + p.sd) % p.Dp, y = (ph + p.sh) % p.Hp, x = (pw + p.sw) % p.Wp;   // position before the roll
      if (d < p.D && y < p.H && x < p.W) t = ((b * p.D + d) * p.H + y) * p.W + x;
      // compute_mask: three slices per dimension, (0, -w), (-w, -s), (-s, end); a zero shift leaves one region
      const int rd = p.sd == 0 ? 2 : (pd < p.Dp - p.wd ? 0 : (pd < p.Dp - p.sd ? 1 : 2));
      const int rh = p.sh == 0 ? 2 : (ph < p.Hp - p.wh ? 0 : (ph < p.Hp - p.sh ? 1 : 2));
      const int rw = p.sw == 0 ? 2 : (pw < p.Wp - p.ww ? 0 : (pw < p.Wp - p.sw ? 1 : 2));
      l = rd * 9 + rh * 3 + rw;
    }
    tok[i] = t;
    lab[i] = l;
  }
  __syncthreads();
  {
    constexpr int CH = HD / 8;                                  // 16-byte chunks per head row
    for (int i = threadIdx.x; i < p.NP * CH * 3; i += 256) {
      const int which = i / (p.NP * CH), j = i - which * p.NP * CH;
      const int row = j / CH, c = j - row * CH;
      uint4 v = make_uint4(0, 0, 0, 0);
      if (row < p.N) {
        const int col = which * p.C + h * HD + c * 8;
        if (tok[row] >= 0) v = *reinterpret_cast<const uint4*>(p.qkv + (size_t)tok[row] * p.ldqkv + col);
        else if (p.pad_qkv != nullptr) v = *reinterpret_cast<const uint4*>(p.pad_qkv + col);
      }
      __nv_bfloat16* dst = (which == 0 ? qs : which == 1 ? ks : vs) + (size_t)row * LDS + c * 8;
      *reinterpret_cast<uint4*>(dst) = v;
    }
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t4 = lane & 3;
  const float scale = rsqrtf((float)HD);
  constexpr float LOG2E = 1.4426950408889634f;
  constexpr int NTMAX = W3_MAXNP / 8;
  const int NT = p.NP / 8;
  for (int mt = warp; mt * 16 < p.N; mt += 8) {
    const int r0 = mt * 16 + g, r1 = r0 + 8;
    float s[NTMAX][4];
#pragma unroll
    for (int nt = 0; nt < NTMAX; ++nt) { s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f; }
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk) {
      uint32_t a[4];
      a[0] = *reinterpret_cast<const uint32_t*>(qs + (size_t)r0 * LDS + kk * 16 + 2 * t4);
      a[1] = *reinterpret_cast<const uint32_t*>(qs + (size_t)r1 * LDS + kk * 16 + 2 * t4);
      a[2] = *reinterpret_cast<const uint32_t*>(qs + (size_t)r0 * LDS + kk * 16 + 8 + 2 * t4);
      a[3] = *reinterpret_cast<const uint32_t*>(qs + (size_t)r1 * LDS + kk * 16 + 8 + 2 * t4);
#pragma unroll
      for (int nt = 0; nt < NTMAX; ++nt) {
        if (nt < NT) {
          const __nv_bfloat16* kr = ks + (size_t)(nt * 8 + g) * LDS + kk * 16 + 2 * t4;
          w3_mma_16816(s[nt], a, *reinterpret_cast<const uint32_t*>(kr), *reinterpret_cast<const uint32_t*>(kr + 8));
        }
      }
    }
    const int q0 = r0 < p.N ? r0 : p.N - 1, q1 = r1 < p.N ? r1 : p.N - 1;      // clamp the bias row of padding rows
    const float* b0p = p.bias + ((size_t)h * p.N + q0) * p.N;
    const float* b1p = p.bias + ((size_t)h * p.N + q1) * p.N;
    const int l0 = lab[q0], l1 = lab[q1];
    float m0 = -1e30f, m1 = -1e30f;
#pragma unroll
    for (int nt = 0; nt < NTMAX; ++nt) {
      if (nt < NT) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int c = nt * 8 + 2 * t4 + e;
          if (c < p.N) {
            float v0 = s[nt][e] * scale + __ldg(b0p + c), v1 = s[nt][2 + e] * scale + __ldg(b1p + c);
            if (shifted) {
              const int lc = lab[c];
              if (lc != l0) v0 += -100.f;
              if (lc != l1) v1 += -100.f;
            }
            s[nt][e] = v0; s[nt][2 + e] = v1;
            m0 = fmaxf(m0, v0); m1 = fmaxf(m1, v1);
          } else {
            s[nt][e] = -1e30f; s[nt][2 + e] = -1e30f;                     // columns beyond the window: no weight
          }
        }
      }
    }
    m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 1)); m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 2));
    m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 1)); m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 2));
    float sum0 = 0.f, sum1 = 0.f;
#pragma unroll
    for (int nt = 0; nt < NTMAX; ++nt) {
      if (nt < NT) {
        s[nt][0] = exp2f((s[nt][0] - m0) * LOG2E); s[nt][1] = exp2f((s[nt][1] - m0) * LOG2E);
        s[nt][2] = exp2f((s[nt][2] - m1) * LOG2E); s[nt][3] = exp2f((s[nt][3] - m1) * LOG2E);
        sum0 += s[nt][0] + s[nt][1];
        sum1 += s[nt][2] + s[nt][3];
      }
    }
    sum0 += __shfl_xor_sync(0xffffffffu, sum0, 1); sum0 += __shfl_xor_sync(0xffffffffu, sum0, 2);
    sum1 += __shfl_xor_sync(0xffffffffu, sum1, 1); sum1 += __shfl_xor_sync(0xffffffffu, sum1, 2);
    const float inv0 = 1.f / sum0, inv1 = 1.f / sum1;
    float o[HD / 8][4];
#pragma unroll
    for (int nt = 0; nt < HD / 8; ++nt) { o[nt][0] = o[nt][1] = o[nt][2] = o[nt][3] = 0.f; }
#pragma unroll
    for (int kk = 0; kk < NTMAX / 2; ++kk) {
      if (2 * kk < NT) {
        uint32_t a[4];
        a[0] = pack_bf16x2(s[2 * kk][0] * inv0, s[2 * kk][1] * inv0);
        a[1] = pack_bf16x2(s[2 * kk][2] * inv1, s[2 * kk][3] * inv1);
        a[2] = pack_bf16x2(s[2 * kk + 1][0] * inv0, s[2 * kk + 1][1] * inv0);
        a[3] = pack_bf16x2(s[2 * kk + 1][2] * inv1, s[2 * kk + 1][3] * inv1);
#pragma unroll
        for (int nt = 0; nt < HD / 8; ++nt) {
          uint32_t b0, b1;
          w3_ldmatrix_x2_trans(b0, b1, vs + (size_t)(kk * 16 + (lane & 15)) * LDS + nt * 8);
          w3_mma_16816(o[nt], a, b0, b1);
        }
      }
    }
    // window_reverse + roll back + crop: rows of real tokens go back to their own position, padding rows are dropped
    if (r0 < p.N && tok[r0] >= 0) {
      __nv_bfloat16* dst = p.out + (size_t)tok[r0] * p.ldo + h * HD;
#pragma unroll
      for (int nt = 0; nt < HD / 8; ++nt) *reinterpret_cast<uint32_t*>(dst + nt * 8 + 2 * t4) = pack_bf16x2(o[nt][0], o[nt][1]);
    }
    if (r1 < p.N && tok[r1] >= 0) {
      __nv_bfloat16* dst = p.out + (size_t)tok[r1] * p.ldo + h * HD;
#pragma unroll
      for (int nt = 0; nt < HD / 8; ++nt) *reinterpret_cast<uint32_t*>(dst + nt * 8 + 2 * t4) = pack_bf16x2(o[nt][2], o[nt][3]);
    }
  }
}

}  // namespace pgt

using namespace pgt;

extern "C" int pgt_window3d_attention(const void* qkv, int ldqkv, const void* pad_qkv, int B, int D, int H, int W, int C,
                                      int heads, int wd, int wh, int ww, int sd, int sh, int sw, const float* bias,
                                      void* out, int ldo, void* stream) {
  PGT_CHECK_ARG(qkv && bias && out && B > 0 && D > 0 && H > 0 && W > 0 && heads > 0 && C % heads == 0);
  PGT_CHECK_ARG(wd > 0 && wh > 0 && ww > 0 && sd >= 0 && sh >= 0 && sw >= 0 && ldqkv % 8 == 0 && ldo % 8 == 0 && ldqkv >= 3 * C);
  // get_window_size (modules/swin.py:70-84): a dimension no larger than the window is one window, unshifted
  if (D <= wd) { wd = D; sd = 0; }
  if (H <= wh) { wh = H; sh = 0; }
  if (W <= ww) { ww = W; sw = 0; }
  const int N = wd * wh * ww, hd = C / heads;
  if (N > W3_MAXNP || (hd != 16 && hd != 32 && hd != 64)) return PGT_ERR_UNSUPPORTED;
  PGT_CHECK_ARG(sd < wd && sh < wh && sw < ww);
  Win3dParams p{};
  p.qkv = reinterpret_cast<const __nv_bfloat16*>(qkv); p.ldqkv = ldqkv;
  p.pad_qkv = reinterpret_cast<const __nv_bfloat16*>(pad_qkv);
  p.bias = bias; p.out = reinterpret_cast<__nv_bfloat16*>(out); p.ldo = ldo;
  p.B = B; p.D = D; p.H = H; p.W = W; p.C = C; p.heads = heads;
  p.wd = wd; p.wh = wh; p.ww = ww; p.sd = sd; p.sh = sh; p.sw = sw;
  p.nd = ceil_div(D, wd); p.nh = ceil_div(H, wh); p.nw = ceil_div(W, ww);
  p.Dp = p.nd * wd; p.Hp = p.nh * wh; p.Wp = p.nw * ww;
  p.N = N; p.NP = (N + 15) / 16 * 16;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  dim3 grid(B * p.nd * p.nh * p.nw, heads);
  const size_t smem = (size_t)3 * W3_MAXNP * (hd + 8) * 2;
  ProfScope ps(PGT_PROF_WINDOW_ATTN, 4.0 * N * N * C * (double)grid.x, st, "window3d");
  if (hd == 16) window3d_attn_kernel<16><<<grid, 256, smem, st>>>(p);
  else if (hd == 32) window3d_attn_kernel<32><<<grid, 256, smem, st>>>(p);
  else {
    static PerDeviceOnce once;                      // 55 KB of dynamic shared memory: above the default limit
    PGT_CUDA_OK(once.run([] { return cudaFuncSetAttribute(window3d_attn_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                          3 * W3_MAXNP * (64 + 8) * 2); }));
    window3d_attn_kernel<64><<<grid, 256, smem, st>>>(p);
  }
  PGT_LAUNCH_OK();
  return PGT_OK;
}
