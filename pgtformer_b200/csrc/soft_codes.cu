// Soft codes of the RQ bottleneck (RQBottleneck.get_soft_codes, archs/tdcrqvae3_arch.py:429-457, depth 1):
//
//   p[t, k] = softmax_k(-||z_t - e_k||^2 / temp) = softmax_k((2 z_t.e_k - ||e_k||^2) / temp)
//
// (||z_t||^2 is constant within a row, so it is left out: mathematically the same, one rounding fewer than the
// reference's addmm).  The scores are probabilities after the softmax, so unlike the argmin (l2_argmin_tc.cu, exact
// about WHICH code is nearest from bf16 scores plus a certificate) the dot products themselves must be about as accurate
// as fp32: at temp 1 an error of d in the score is a relative error of d in p.
//
// 3xTF32 on the tensor cores: every fp32 operand x is split into x_hi = tf32(x) and x_lo = tf32(x - x_hi), and
//   z.e ~= z_lo.e_hi + z_hi.e_lo + z_hi.e_hi        (z_lo.e_lo ~ 2^-22 relative, dropped)
// with mma.sync m16n8k8 .tf32 (products are exact in fp32).  The split is done while the fragments are read from
// shared memory, so shared memory holds the raw fp32 tiles once (half the traffic of pre-split hi / lo copies).  The
// tensor core's fp32 accumulation does not round to nearest; to keep that error from building up over E = 512, each
// 32-wide k-chunk is accumulated from zero (12 MMAs per fragment) and then added to an fp32 register total with an
// ordinary round-to-nearest add.
//
// Tiling: 128 tokens x 128 codes per CTA step, k-chunk 32, 3-stage cp.async ring of raw fp32 tiles; 8 warps as
// 2 (tokens) x 4 (codes), each warp 64 x 32 = 4 x 4 fragments.  The CTA walks all K / 128 code tiles of its 128 tokens:
// the epilogue of each code tile writes s = (2 dot - ||e||^2) / temp to the output and updates a per-row online
// (max, sum of exp); after the last tile the CTA merges the row statistics, then re-reads its own rows (L2-resident,
// written by this CTA) and rewrites them in place as exp(s - max) / sum.
#include <float.h>

#include "common.cuh"
#include "ptx.cuh"
#include "tmap.cuh"

namespace pgt {

constexpr int SC_BM = 128;                 // tokens per CTA
constexpr int SC_BN = 128;                 // codes per tile
constexpr int SC_BK = 32;                  // k-chunk
constexpr int SC_LD = SC_BK + 4;           // smem row pitch (floats): fragment reads hit 32 distinct banks
constexpr int SC_ST = 3;                   // cp.async stages
constexpr int SC_STAGE_FLOATS = (SC_BM + SC_BN) * SC_LD;
constexpr int SC_SMEM = SC_ST * SC_STAGE_FLOATS * 4 + 2 * 4 * SC_BM * 4;   // ring + [2][4 warps][128 rows] row stats
static_assert(SC_SMEM <= 232448, "soft_codes smem budget");

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
  // src-size 0 zero-fills the 16 bytes (rows past T)
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hi) : "f"(x));
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(lo) : "f"(x - __uint_as_float(hi)));
}

__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__global__ void __launch_bounds__(256, 1)
soft_codes_kernel(const float* __restrict__ z, int T, int E, const float* __restrict__ cb, const float* __restrict__ norm,
                  int K, float temp, float* __restrict__ out, int ldo) {
  extern __shared__ __align__(16) float sm[];
  float* rstat = sm + SC_ST * SC_STAGE_FLOATS;            // [2][4][128]: per code-warp row max, row sum
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wm = warp >> 2, wn = warp & 3;                // 64-row half, 32-code quarter
  const int g = lane >> 2, tq = lane & 3;
  const int t0 = blockIdx.x * SC_BM;
  const int KC = E / SC_BK, NT = K / SC_BN, total = NT * KC;

  // stage loader: 128 token rows and 128 code rows of one k-chunk, 8 x 16 B per row, 4 + 4 copies per thread
  auto load = [&](int it, int s) {
    const int nt = it / KC, kc = it % KC;
    float* sa = sm + s * SC_STAGE_FLOATS;
    float* sb = sa + SC_BM * SC_LD;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int c = tid + i * 256, r = c >> 3, q = (c & 7) * 4;
      const int t = t0 + r;
      cp_async16(smem_u32(sa + r * SC_LD + q), z + (size_t)(t < T ? t : 0) * E + kc * SC_BK + q, t < T);
      cp_async16(smem_u32(sb + r * SC_LD + q), cb + (size_t)(nt * SC_BN + r) * E + kc * SC_BK + q, true);
    }
  };

#pragma unroll
  for (int s = 0; s < SC_ST - 1; ++s) {
    if (s < total) load(s, s);
    cp_async_commit();
  }

  float acc[4][4][4];                                     // fp32 (round-to-nearest) totals of the current code tile
  float rmax[4][2], rsum[4][2];                           // online row statistics: fragment i, row g / g + 8
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    rmax[i][0] = rmax[i][1] = -FLT_MAX;
    rsum[i][0] = rsum[i][1] = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = acc[i][j][2] = acc[i][j][3] = 0.f;
  }

  for (int it = 0; it < total; ++it) {
    cp_async_wait<SC_ST - 2>();
    __syncthreads();                                      // stage it % ST landed; stage (it - 1) % ST is free
    if (it + SC_ST - 1 < total) load(it + SC_ST - 1, (it + SC_ST - 1) % SC_ST);
    cp_async_commit();

    const float* sa = sm + (it % SC_ST) * SC_STAGE_FLOATS + (wm * 64) * SC_LD;
    const float* sb = sm + (it % SC_ST) * SC_STAGE_FLOATS + SC_BM * SC_LD + (wn * 32) * SC_LD;
    float part[4][4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) part[i][j][0] = part[i][j][1] = part[i][j][2] = part[i][j][3] = 0.f;
#pragma unroll
    for (int k8 = 0; k8 < SC_BK / 8; ++k8) {
      uint32_t ah[4][4], al[4][4], bh[4][2], bl[4][2];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float* p = sa + (16 * i + g) * SC_LD + 8 * k8 + tq;
        split_tf32(p[0], ah[i][0], al[i][0]);
        split_tf32(p[8 * SC_LD], ah[i][1], al[i][1]);
        split_tf32(p[4], ah[i][2], al[i][2]);
        split_tf32(p[8 * SC_LD + 4], ah[i][3], al[i][3]);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float* p = sb + (8 * j + g) * SC_LD + 8 * k8 + tq;
        split_tf32(p[0], bh[j][0], bl[j][0]);
        split_tf32(p[4], bh[j][1], bl[j][1]);
      }
      // small terms first; each pass issues 16 independent MMAs, so no MMA waits on the one before it
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) mma_tf32(part[i][j], al[i], bh[j][0], bh[j][1]);
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) mma_tf32(part[i][j], ah[i], bl[j][0], bl[j][1]);
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) mma_tf32(part[i][j], ah[i], bh[j][0], bh[j][1]);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[i][j][e] += part[i][j][e];

    if ((it % KC) == KC - 1) {
      // ---- epilogue of code tile nt: scores to the output, online row statistics
      const int nt = it / KC;
      float nrm[4][2];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 n2 = __ldg(reinterpret_cast<const float2*>(norm + nt * SC_BN + wn * 32 + 8 * j + 2 * tq));
        nrm[j][0] = n2.x; nrm[j][1] = n2.y;
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int t = t0 + wm * 64 + 16 * i + g + 8 * h;
          float s[8];
          float m = rmax[i][h];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            s[2 * j] = __fdiv_rn(fmaf(2.f, acc[i][j][2 * h], -nrm[j][0]), temp);
            s[2 * j + 1] = __fdiv_rn(fmaf(2.f, acc[i][j][2 * h + 1], -nrm[j][1]), temp);
            m = fmaxf(m, fmaxf(s[2 * j], s[2 * j + 1]));
          }
          float sum = rsum[i][h] * expf(rmax[i][h] - m);
#pragma unroll
          for (int q = 0; q < 8; ++q) sum += expf(s[q] - m);
          rmax[i][h] = m;
          rsum[i][h] = sum;
          if (t < T) {
            float* o = out + (size_t)t * ldo + nt * SC_BN + wn * 32 + 2 * tq;
#pragma unroll
            for (int j = 0; j < 4; ++j) *reinterpret_cast<float2*>(o + 8 * j) = make_float2(s[2 * j], s[2 * j + 1]);
          }
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = acc[i][j][2] = acc[i][j][3] = 0.f;
      }
    }
  }
  cp_async_wait<0>();

  // ---- merge the row statistics: the 4 lanes of a quad, then the 4 code warps
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float m = rmax[i][h], s = rsum[i][h];
#pragma unroll
      for (int o = 1; o <= 2; o <<= 1) {
        const float om = __shfl_xor_sync(0xffffffffu, m, o), os = __shfl_xor_sync(0xffffffffu, s, o);
        const float nm = fmaxf(m, om);
        s = s * expf(m - nm) + os * expf(om - nm);
        m = nm;
      }
      if (tq == 0) {
        const int r = wm * 64 + 16 * i + g + 8 * h;
        rstat[wn * SC_BM + r] = m;
        rstat[4 * SC_BM + wn * SC_BM + r] = s;
      }
    }
  __syncthreads();                                        // also orders this CTA's score stores before the re-reads

  // ---- rewrite the CTA's rows in place: p = exp(s - max) / sum (one warp per row, float4 streams)
  for (int r = warp; r < SC_BM; r += 8) {
    const int t = t0 + r;
    if (t >= T) break;
    float m = -FLT_MAX;
#pragma unroll
    for (int w = 0; w < 4; ++w) m = fmaxf(m, rstat[w * SC_BM + r]);
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 4; ++w) s += rstat[4 * SC_BM + w * SC_BM + r] * expf(rstat[w * SC_BM + r] - m);
    float4* row = reinterpret_cast<float4*>(out + (size_t)t * ldo);
    for (int c = lane; c < (K >> 2); c += 32) {
      float4 v = row[c];
      v.x = __fdiv_rn(expf(v.x - m), s);
      v.y = __fdiv_rn(expf(v.y - m), s);
      v.z = __fdiv_rn(expf(v.z - m), s);
      v.w = __fdiv_rn(expf(v.w - m), s);
      row[c] = v;
    }
  }
}

}  // namespace pgt

using namespace pgt;

extern "C" int pgt_soft_codes(const float* z, int T, int E, const float* codebook, const float* cb_norm, int K, float temp,
                              float* out, int ldo, void* stream) {
  PGT_CHECK_ARG(z && codebook && cb_norm && out && T > 0 && K > 0 && E > 0 && ldo >= K && ldo % 4 == 0);
  PGT_CHECK_ARG(temp > 0.f && temp <= FLT_MAX);            // also rejects NaN
  PGT_CHECK_ARG((reinterpret_cast<uintptr_t>(z) & 15) == 0 && (reinterpret_cast<uintptr_t>(codebook) & 15) == 0 &&
                (reinterpret_cast<uintptr_t>(out) & 15) == 0 && (reinterpret_cast<uintptr_t>(cb_norm) & 7) == 0);
  if (K % SC_BN != 0 || E % SC_BK != 0) return PGT_ERR_UNSUPPORTED;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  static PerDeviceOnce once;
  PGT_CUDA_OK(once.run([] { return cudaFuncSetAttribute(soft_codes_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SC_SMEM); }));
  ProfScope ps(PGT_PROF_ARGMIN, 2.0 * T * (double)K * E, st, "soft_codes");
  soft_codes_kernel<<<ceil_div(T, SC_BM), 256, SC_SMEM, st>>>(z, T, E, codebook, cb_norm, K, temp, out, ldo);
  PGT_LAUNCH_OK();
  return PGT_OK;
}
