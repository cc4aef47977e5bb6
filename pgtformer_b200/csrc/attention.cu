// Attention cores (round-1 implementation on the warp-level mma.sync path; the wgmma fused
// Swin-block kernel replaces the window kernel in a later round — see DESIGN.md):
//   * shifted-window spatio-temporal attention, 3x4x4 windows (N = 48), roll / partition / reverse and the
//     {0,-100} shift mask done as index math, relative-position bias from a [heads,48,48] table;
//   * global multi-head flash attention (online softmax, K/V tiles double-buffered with cp.async).
#include <cstdlib>

#include "common.cuh"

namespace pgt {

__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void ldmatrix_x2_trans(uint32_t& r0, uint32_t& r1, const void* smem_row_ptr) {
  const uint32_t a = static_cast<uint32_t>(__cvta_generic_to_shared(smem_row_ptr));
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0,%1}, [%2];" : "=r"(r0), "=r"(r1) : "r"(a));
}
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc, bool pred) {
  const uint32_t d = static_cast<uint32_t>(__cvta_generic_to_shared(smem_dst));
  const int sz = pred ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(gsrc), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// =============================================================================== window attention
// CTA = one 3x4x4 window (48 tokens).  The tokens' full [q | k | v] rows (3C bf16, contiguous in HBM) are staged
// into shared memory with coalesced 16-byte cp.async copies; warp h then runs head h entirely out of smem
// (QK^T and PV on mma.sync m16n8k16, fp32 softmax with the relative-position bias and the {0,-100} shift mask),
// overwrites its own q columns with the result, and the CTA streams the 48 x C output rows back coalesced.
constexpr int WIN_N = 48;

template <int D>
__global__ void __launch_bounds__(256)
window_attn_kernel(const __nv_bfloat16* __restrict__ qkv, int ldqkv, int H, int W, int C, int heads, int sy, int sx,
                   const float* __restrict__ bias_tab, __nv_bfloat16* __restrict__ out, int ldo) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ int tok[WIN_N];
  __shared__ int lab[WIN_N];
  const int LDR = 3 * C + 8;                               // padded smem row (bf16 elements): stride = 4 words mod 32
  __nv_bfloat16* rows = reinterpret_cast<__nv_bfloat16*>(smem_raw);
  const int nwx = W >> 2;
  const int wx = blockIdx.x % nwx, wy = blockIdx.x / nwx, clip = blockIdx.y;
  if (threadIdx.x < WIN_N) {
    const int i = threadIdx.x;
    const int fr = i >> 4, iy = (i >> 2) & 3, ix = i & 3;
    const int ys = wy * 4 + iy, xs = wx * 4 + ix;         // coordinates in the rolled (shifted) frame
    const int y = (ys + sy) % H, x = (xs + sx) % W;       // source / destination pixel (roll by -shift, then back)
    tok[i] = ((clip * 3 + fr) * H + y) * W + x;
    const int hr = ys < H - 4 ? 0 : (ys < H - sy ? 1 : 2); // an unshifted axis is one region
    const int wr = xs < W - 4 ? 0 : (xs < W - sx ? 1 : 2);
    lab[i] = hr * 3 + wr;
  }
  __syncthreads();
  {
    const int chunks = (3 * C) >> 3;                       // 16-byte chunks per token row
    for (int i = threadIdx.x; i < WIN_N * chunks; i += 256) {
      const int r = i / chunks, c = i - r * chunks;
      cp_async16(rows + (size_t)r * LDR + c * 8, qkv + (size_t)tok[r] * ldqkv + c * 8, true);
    }
    cp_async_commit();
    cp_async_wait<0>();
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const float scale = rsqrtf((float)D);
  constexpr float LOG2E = 1.4426950408889634f;

  for (int h = warp; h < heads; h += 8) {
    const __nv_bfloat16* qs = rows + h * D;
    const __nv_bfloat16* ks = rows + C + h * D;
    const __nv_bfloat16* vs = rows + 2 * C + h * D;
    for (int mt = 0; mt < 3; ++mt) {
      float o[D / 8][4];
      const int r0 = mt * 16 + g, r1 = r0 + 8;
      float s[6][4];
#pragma unroll
      for (int nt = 0; nt < 6; ++nt) { s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f; }
#pragma unroll
      for (int kk = 0; kk < D / 16; ++kk) {
        uint32_t a[4];
        a[0] = *reinterpret_cast<const uint32_t*>(qs + (size_t)r0 * LDR + kk * 16 + 2 * t);
        a[1] = *reinterpret_cast<const uint32_t*>(qs + (size_t)r1 * LDR + kk * 16 + 2 * t);
        a[2] = *reinterpret_cast<const uint32_t*>(qs + (size_t)r0 * LDR + kk * 16 + 8 + 2 * t);
        a[3] = *reinterpret_cast<const uint32_t*>(qs + (size_t)r1 * LDR + kk * 16 + 8 + 2 * t);
#pragma unroll
        for (int nt = 0; nt < 6; ++nt) {
          const __nv_bfloat16* kr = ks + (size_t)(nt * 8 + g) * LDR + kk * 16 + 2 * t;
          mma_bf16_16816(s[nt], a, *reinterpret_cast<const uint32_t*>(kr), *reinterpret_cast<const uint32_t*>(kr + 8));
        }
      }
      // scale, + relative-position bias, + shift mask; fp32 softmax over the 48 keys of each row
      const float* b0p = bias_tab + ((size_t)h * WIN_N + r0) * WIN_N;
      const float* b1p = bias_tab + ((size_t)h * WIN_N + r1) * WIN_N;
      const int l0 = lab[r0], l1 = lab[r1];
      float m0 = -1e30f, m1 = -1e30f;
#pragma unroll
      for (int nt = 0; nt < 6; ++nt) {
        const int c = nt * 8 + 2 * t;
        const float2 bb0 = __ldg(reinterpret_cast<const float2*>(b0p + c));
        const float2 bb1 = __ldg(reinterpret_cast<const float2*>(b1p + c));
        s[nt][0] = s[nt][0] * scale + bb0.x;
        s[nt][1] = s[nt][1] * scale + bb0.y;
        s[nt][2] = s[nt][2] * scale + bb1.x;
        s[nt][3] = s[nt][3] * scale + bb1.y;
        if (sy > 0 || sx > 0) {
          const int lc0 = lab[c], lc1 = lab[c + 1];
          if (lc0 != l0) s[nt][0] += -100.f;
          if (lc1 != l0) s[nt][1] += -100.f;
          if (lc0 != l1) s[nt][2] += -100.f;
          if (lc1 != l1) s[nt][3] += -100.f;
        }
        m0 = fmaxf(m0, fmaxf(s[nt][0], s[nt][1]));
        m1 = fmaxf(m1, fmaxf(s[nt][2], s[nt][3]));
      }
      m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 1)); m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 2));
      m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 1)); m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 2));
      float sum0 = 0.f, sum1 = 0.f;
#pragma unroll
      for (int nt = 0; nt < 6; ++nt) {
        s[nt][0] = exp2f((s[nt][0] - m0) * LOG2E); s[nt][1] = exp2f((s[nt][1] - m0) * LOG2E);
        s[nt][2] = exp2f((s[nt][2] - m1) * LOG2E); s[nt][3] = exp2f((s[nt][3] - m1) * LOG2E);
        sum0 += s[nt][0] + s[nt][1];
        sum1 += s[nt][2] + s[nt][3];
      }
      sum0 += __shfl_xor_sync(0xffffffffu, sum0, 1); sum0 += __shfl_xor_sync(0xffffffffu, sum0, 2);
      sum1 += __shfl_xor_sync(0xffffffffu, sum1, 1); sum1 += __shfl_xor_sync(0xffffffffu, sum1, 2);
      const float inv0 = 1.f / sum0, inv1 = 1.f / sum1;
      // O = P V  (P normalised in fp32 before the bf16 pack, as the reference's softmax output is)
#pragma unroll
      for (int nt = 0; nt < D / 8; ++nt) { o[nt][0] = o[nt][1] = o[nt][2] = o[nt][3] = 0.f; }
#pragma unroll
      for (int kk = 0; kk < 3; ++kk) {
        uint32_t a[4];
        a[0] = pack_bf16x2(s[2 * kk][0] * inv0, s[2 * kk][1] * inv0);
        a[1] = pack_bf16x2(s[2 * kk][2] * inv1, s[2 * kk][3] * inv1);
        a[2] = pack_bf16x2(s[2 * kk + 1][0] * inv0, s[2 * kk + 1][1] * inv0);
        a[3] = pack_bf16x2(s[2 * kk + 1][2] * inv1, s[2 * kk + 1][3] * inv1);
#pragma unroll
        for (int nt = 0; nt < D / 8; ++nt) {
          uint32_t b0, b1;
          ldmatrix_x2_trans(b0, b1, vs + (size_t)(kk * 16 + (lane & 15)) * LDR + nt * 8);
          mma_bf16_16816(o[nt], a, b0, b1);
        }
      }
      // only this row tile reads q rows [mt*16, mt*16+16) of head h: overwrite them with the head's output
      __syncwarp();
      __nv_bfloat16* o0 = rows + (size_t)r0 * LDR + h * D;
      __nv_bfloat16* o1 = rows + (size_t)r1 * LDR + h * D;
#pragma unroll
      for (int nt = 0; nt < D / 8; ++nt) {
        *reinterpret_cast<uint32_t*>(o0 + nt * 8 + 2 * t) = pack_bf16x2(o[nt][0], o[nt][1]);
        *reinterpret_cast<uint32_t*>(o1 + nt * 8 + 2 * t) = pack_bf16x2(o[nt][2], o[nt][3]);
      }
    }
  }
  __syncthreads();
  {
    const int chunks = C >> 3;                             // 16-byte chunks per output row
    for (int i = threadIdx.x; i < WIN_N * chunks; i += 256) {
      const int r = i / chunks, c = i - r * chunks;
      *reinterpret_cast<uint4*>(out + (size_t)tok[r] * ldo + c * 8) = *reinterpret_cast<const uint4*>(rows + (size_t)r * LDR + c * 8);
    }
  }
}

// =============================================================================== global flash attention
constexpr int FA_BM = 64;     // queries per CTA (4 warps x 16 rows)
constexpr int FA_BN = 64;     // keys per tile

template <int D>
__global__ void __launch_bounds__(128)
mha_fwd_kernel(const __nv_bfloat16* __restrict__ q, int ldq, const __nv_bfloat16* __restrict__ k, int ldk,
               const __nv_bfloat16* __restrict__ v, int ldv, int L, int heads, __nv_bfloat16* __restrict__ out, int ldo) {
  constexpr int LDS = D + 8;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __nv_bfloat16* ks = reinterpret_cast<__nv_bfloat16*>(smem_raw);          // [2][FA_BN][LDS]
  __nv_bfloat16* vs = ks + 2 * FA_BN * LDS;                                // [2][FA_BN][LDS]
  const int qt = blockIdx.x, h = blockIdx.y, clip = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const size_t row_base = (size_t)clip * L;
  const __nv_bfloat16* kbase = k + row_base * ldk + h * D;
  const __nv_bfloat16* vbase = v + row_base * ldv + h * D;
  const int ntiles = (L + FA_BN - 1) / FA_BN;
  constexpr int CH = D / 8;

  auto load_tile = [&](int tile, int buf) {
    for (int i = threadIdx.x; i < FA_BN * CH; i += 128) {
      const int r = i / CH, c = i % CH;
      const int key = tile * FA_BN + r;
      const bool ok = key < L;
      const size_t kr = ok ? key : 0;
      cp_async16(ks + ((size_t)buf * FA_BN + r) * LDS + c * 8, kbase + kr * ldk + c * 8, ok);
      cp_async16(vs + ((size_t)buf * FA_BN + r) * LDS + c * 8, vbase + kr * ldv + c * 8, ok);
    }
  };
  load_tile(0, 0);
  cp_async_commit();

  // Q fragments (16 rows x D) straight from global
  const int qr0 = qt * FA_BM + warp * 16 + g, qr1 = qr0 + 8;
  const bool v0 = qr0 < L, v1 = qr1 < L;
  const __nv_bfloat16* q0 = q + (row_base + (v0 ? qr0 : 0)) * ldq + h * D;
  const __nv_bfloat16* q1 = q + (row_base + (v1 ? qr1 : 0)) * ldq + h * D;
  uint32_t qa[D / 16][4];
#pragma unroll
  for (int kk = 0; kk < D / 16; ++kk) {
    qa[kk][0] = v0 ? __ldg(reinterpret_cast<const uint32_t*>(q0 + kk * 16 + 2 * t)) : 0u;
    qa[kk][1] = v1 ? __ldg(reinterpret_cast<const uint32_t*>(q1 + kk * 16 + 2 * t)) : 0u;
    qa[kk][2] = v0 ? __ldg(reinterpret_cast<const uint32_t*>(q0 + kk * 16 + 8 + 2 * t)) : 0u;
    qa[kk][3] = v1 ? __ldg(reinterpret_cast<const uint32_t*>(q1 + kk * 16 + 8 + 2 * t)) : 0u;
  }
  const float sl2 = rsqrtf((float)D) * 1.4426950408889634f;     // softmax scale in the log2 domain
  float m0 = -1e30f, m1 = -1e30f, l0 = 0.f, l1 = 0.f;
  float o[D / 8][4];
#pragma unroll
  for (int nt = 0; nt < D / 8; ++nt) { o[nt][0] = o[nt][1] = o[nt][2] = o[nt][3] = 0.f; }

  for (int tile = 0; tile < ntiles; ++tile) {
    const int buf = tile & 1;
    if (tile + 1 < ntiles) load_tile(tile + 1, buf ^ 1);
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    const __nv_bfloat16* kt = ks + (size_t)buf * FA_BN * LDS;
    const __nv_bfloat16* vt = vs + (size_t)buf * FA_BN * LDS;
    float s[FA_BN / 8][4];
#pragma unroll
    for (int nt = 0; nt < FA_BN / 8; ++nt) { s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f; }
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) {
#pragma unroll
      for (int nt = 0; nt < FA_BN / 8; ++nt) {
        const __nv_bfloat16* kr = kt + (nt * 8 + g) * LDS + kk * 16 + 2 * t;
        mma_bf16_16816(s[nt], qa[kk], *reinterpret_cast<const uint32_t*>(kr), *reinterpret_cast<const uint32_t*>(kr + 8));
      }
    }
    const bool tail = (tile + 1) * FA_BN > L;
    float mx0 = m0, mx1 = m1;
#pragma unroll
    for (int nt = 0; nt < FA_BN / 8; ++nt) {
      if (tail) {
        const int c = tile * FA_BN + nt * 8 + 2 * t;
        if (c >= L) { s[nt][0] = -1e30f; s[nt][2] = -1e30f; }
        if (c + 1 >= L) { s[nt][1] = -1e30f; s[nt][3] = -1e30f; }
      }
      mx0 = fmaxf(mx0, fmaxf(s[nt][0], s[nt][1]));
      mx1 = fmaxf(mx1, fmaxf(s[nt][2], s[nt][3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float c0 = exp2f((m0 - mx0) * sl2), c1 = exp2f((m1 - mx1) * sl2);
    m0 = mx0; m1 = mx1;
    float rs0 = 0.f, rs1 = 0.f;
#pragma unroll
    for (int nt = 0; nt < FA_BN / 8; ++nt) {
      s[nt][0] = exp2f((s[nt][0] - m0) * sl2); s[nt][1] = exp2f((s[nt][1] - m0) * sl2);
      s[nt][2] = exp2f((s[nt][2] - m1) * sl2); s[nt][3] = exp2f((s[nt][3] - m1) * sl2);
      rs0 += s[nt][0] + s[nt][1];
      rs1 += s[nt][2] + s[nt][3];
    }
    l0 = l0 * c0 + rs0;
    l1 = l1 * c1 + rs1;
#pragma unroll
    for (int nt = 0; nt < D / 8; ++nt) { o[nt][0] *= c0; o[nt][1] *= c0; o[nt][2] *= c1; o[nt][3] *= c1; }
#pragma unroll
    for (int kk = 0; kk < FA_BN / 16; ++kk) {
      uint32_t a[4];
      a[0] = pack_bf16x2(s[2 * kk][0], s[2 * kk][1]);
      a[1] = pack_bf16x2(s[2 * kk][2], s[2 * kk][3]);
      a[2] = pack_bf16x2(s[2 * kk + 1][0], s[2 * kk + 1][1]);
      a[3] = pack_bf16x2(s[2 * kk + 1][2], s[2 * kk + 1][3]);
#pragma unroll
      for (int nt = 0; nt < D / 8; ++nt) {
        uint32_t b0, b1;
        ldmatrix_x2_trans(b0, b1, vt + (kk * 16 + (lane & 15)) * LDS + nt * 8);
        mma_bf16_16816(o[nt], a, b0, b1);
      }
    }
    __syncthreads();          // everyone is done with `buf` before the next prefetch overwrites it
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float i0 = 1.f / l0, i1 = 1.f / l1;
  __nv_bfloat16* o0 = out + (row_base + qr0) * ldo + h * D;
  __nv_bfloat16* o1 = out + (row_base + qr1) * ldo + h * D;
#pragma unroll
  for (int nt = 0; nt < D / 8; ++nt) {
    if (v0) *reinterpret_cast<uint32_t*>(o0 + nt * 8 + 2 * t) = pack_bf16x2(o[nt][0] * i0, o[nt][1] * i0);
    if (v1) *reinterpret_cast<uint32_t*>(o1 + nt * 8 + 2 * t) = pack_bf16x2(o[nt][2] * i1, o[nt][3] * i1);
  }
}

int mha_tc_launch(const void* q, int ldq, const void* k, int ldk, const void* v, int ldv, int clips, int L, int heads,
                  int d, void* out, int ldo, cudaStream_t stream);      // mha_tc.cu (wgmma path)
int attn_wide_launch(const void* q, int ldq, const void* k, int ldk, const void* v, int ldv, int clips, int L, int heads,
                     int d, void* out, int ldo, cudaStream_t stream);   // attn_wide_tc.cu (d = 256 / 512)

}  // namespace pgt

using namespace pgt;

extern "C" int pgt_window_attention(const void* qkv, int ldqkv, int clips, int H, int W, int C, int heads, int shift,
                                    const float* bias_tab, void* out, int ldo, void* stream) {
  PGT_CHECK_ARG(qkv && bias_tab && out && clips > 0 && H > 0 && W > 0 && heads > 0);
  PGT_CHECK_ARG(H % 4 == 0 && W % 4 == 0 && C % heads == 0 && ldqkv % 8 == 0 && ldo % 8 == 0 && ldqkv >= 3 * C);
  PGT_CHECK_ARG(shift >= 0 && shift < 4);
  // get_window_size(), per axis: an axis that is one window deep is not shifted, whatever the other axis is
  const int sy = H > 4 ? shift : 0, sx = W > 4 ? shift : 0;
  const int d = C / heads;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  dim3 grid((H / 4) * (W / 4), clips);
  const size_t smem = (size_t)WIN_N * (3 * C + 8) * 2;
  ProfScope ps(PGT_PROF_WINDOW_ATTN, 4.0 * WIN_N * WIN_N * C * (double)grid.x * grid.y, st);
  if (d == 32) {
    static bool attr32 = false;
    if (!attr32) {
      PGT_CUDA_OK(cudaFuncSetAttribute(window_attn_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      attr32 = true;
    }
    window_attn_kernel<32><<<grid, 256, smem, st>>>(reinterpret_cast<const __nv_bfloat16*>(qkv), ldqkv, H, W, C, heads,
                                                    sy, sx, bias_tab, reinterpret_cast<__nv_bfloat16*>(out), ldo);
  } else if (d == 64) {
    static bool attr = false;
    if (!attr) {
      PGT_CUDA_OK(cudaFuncSetAttribute(window_attn_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      attr = true;
    }
    window_attn_kernel<64><<<grid, 256, smem, st>>>(reinterpret_cast<const __nv_bfloat16*>(qkv), ldqkv, H, W, C, heads,
                                                    sy, sx, bias_tab, reinterpret_cast<__nv_bfloat16*>(out), ldo);
  } else {
    return PGT_ERR_UNSUPPORTED;
  }
  PGT_LAUNCH_OK();
  return PGT_OK;
}

extern "C" int pgt_mha_fwd(const void* q, int ldq, const void* k, int ldk, const void* v, int ldv, int clips, int L,
                           int heads, int d, void* out, int ldo, void* stream) {
  PGT_CHECK_ARG(q && k && v && out && clips > 0 && L > 0 && heads > 0);
  PGT_CHECK_ARG(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0);
  if (d == 256 || d == 512) {                        // wide heads: the wgmma kernel is the only path
    ProfScope pst(PGT_PROF_MHA, 4.0 * (double)L * L * d * heads * clips, static_cast<cudaStream_t>(stream), "mha_wide");
    return attn_wide_launch(q, ldq, k, ldk, v, ldv, clips, L, heads, d, out, ldo, static_cast<cudaStream_t>(stream));
  }
  if (d != 64) return PGT_ERR_UNSUPPORTED;
  static const bool no_tc = getenv("PGT_MHA_NO_TC") != nullptr;
  if (!no_tc) {
    ProfScope pst(PGT_PROF_MHA, 4.0 * (double)L * L * d * heads * clips, static_cast<cudaStream_t>(stream), "mha_tc");
    const int rc = mha_tc_launch(q, ldq, k, ldk, v, ldv, clips, L, heads, d, out, ldo, static_cast<cudaStream_t>(stream));
    if (rc != PGT_ERR_UNSUPPORTED) return rc;        // shapes the wgmma kernel does not cover use the mma.sync kernel
  }
  dim3 grid(ceil_div(L, FA_BM), heads, clips);
  const size_t smem = (size_t)4 * FA_BN * (64 + 8) * 2;
  ProfScope ps(PGT_PROF_MHA, 4.0 * (double)L * L * d * heads * clips, static_cast<cudaStream_t>(stream));
  mha_fwd_kernel<64><<<grid, 128, smem, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(q), ldq, reinterpret_cast<const __nv_bfloat16*>(k), ldk,
      reinterpret_cast<const __nv_bfloat16*>(v), ldv, L, heads, reinterpret_cast<__nv_bfloat16*>(out), ldo);
  PGT_LAUNCH_OK();
  return PGT_OK;
}
