// VectorQuantizer.forward of VQGAN / CodeFormer (`archs/vqgan_arch.py:42-84`) after the exact nearest-code argmin
// (pgt_l2_argmin_tc on the fp32 encoder output): everything the module returns besides the codes, without ever forming
// the [T, K] distance matrix.
//   vq_token_kernel: one warp per token t with code c = idx[t], e = codebook[c]:
//     * the straight-through z + (e - z) with one rounding per operation (no FMA contraction), written fp32 NCHW
//       (the code_only return, z_q.permute(0, 3, 1, 2)) and / or bf16 NHWC (the generator's conv_in input);
//     * the one-hot row of min_encodings and min_encoding_scores = exp(-d / 10), d = |z|^2 + |e|^2 - 2 z.e accumulated
//       in fp64 and rounded to fp32 once;
//     * the code counts, added to the module's int32 `usage` buffer and to this call's histogram;
//     * per-block partial sums (fp64) of sum_t z_t [E], sum_t |z_t|^2 and sum_t |e_c - z_t|^2, each warp owning its
//       lanes' columns in shared memory and the block summing its warps in a fixed order: no floating-point atomics,
//       so the scalars are the same bits on every run.
//   vq_finish_kernel (one block): sums the block partials in block order and finishes on the device
//     loss          = m + beta m,  m = sum |e - z|^2 / (T E)
//     perplexity    = exp(-sum_k p_k log(p_k + 1e-10)),  p_k = count_k / T
//     mean_distance = (K sum_t |z_t|^2 + T sum_k |e_k|^2 - 2 (sum_t z_t).(sum_k e_k)) / (T K)    (= mean(d) over [T, K])
#include <cstdio>

#include "common.cuh"

namespace pgt {

constexpr int VQ_WARPS = 8;
constexpr int VQ_MAX_E = 512;
constexpr int VQ_FIN_THREADS = 1024;

static int vq_grid(int T) {
  const int need = (T + VQ_WARPS - 1) / VQ_WARPS;
  return need < 2 * num_sms() ? need : 2 * num_sms();
}

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void __launch_bounds__(VQ_WARPS * 32)
vq_token_kernel(const float* __restrict__ z, int T, int E, int HW, const float* __restrict__ cb, int K,
                const int64_t* __restrict__ idx, float* __restrict__ zq_nchw, __nv_bfloat16* __restrict__ zq_bf16,
                float* __restrict__ min_enc, float* __restrict__ scores, int* __restrict__ usage, int* __restrict__ hist,
                double* __restrict__ ws) {
  __shared__ double sz[VQ_WARPS][VQ_MAX_E];                  // per-warp sum_t z_t, column j owned by lane j % 32
  __shared__ double stot[VQ_WARPS][2];                       // per-warp sum |z|^2, sum |e - z|^2
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int j = lane; j < E; j += 32) sz[warp][j] = 0.0;
  double wzz = 0.0, wsq = 0.0;
  for (int t = blockIdx.x * VQ_WARPS + warp; t < T; t += gridDim.x * VQ_WARPS) {
    const int64_t c = idx[t];
    const float* zr = z + (size_t)t * E;
    const float* er = cb + (size_t)c * E;
    const int bi = t / HW, p = t - bi * HW;
    double zz = 0.0, ee = 0.0, ze = 0.0, sq = 0.0;
    for (int j = lane; j < E; j += 32) {
      const float zj = zr[j], ej = __ldg(er + j);
      const float diff = __fsub_rn(ej, zj);
      const float q = __fadd_rn(zj, diff);
      if (zq_nchw != nullptr) zq_nchw[((size_t)bi * E + j) * HW + p] = q;
      if (zq_bf16 != nullptr) zq_bf16[(size_t)t * E + j] = __float2bfloat16_rn(q);
      zz += (double)zj * zj;
      ee += (double)ej * ej;
      ze += (double)zj * ej;
      sq += (double)diff * diff;
      sz[warp][j] += zj;
    }
    zz = warp_sum_d(zz);
    ee = warp_sum_d(ee);
    ze = warp_sum_d(ze);
    sq = warp_sum_d(sq);
    wzz += zz;
    wsq += sq;
    if (lane == 0) {
      const float d = (float)(zz + ee - 2.0 * ze);
      if (scores != nullptr) scores[t] = (float)exp(-(double)d / 10.0);
      if (usage != nullptr) atomicAdd(usage + c, 1);
      atomicAdd(hist + c, 1);
    }
    if (min_enc != nullptr) {
      float4* row = reinterpret_cast<float4*>(min_enc + (size_t)t * K);
      for (int k4 = lane; k4 < K / 4; k4 += 32) {
        const int k = 4 * k4;
        row[k4] = make_float4(k == c ? 1.f : 0.f, k + 1 == c ? 1.f : 0.f, k + 2 == c ? 1.f : 0.f, k + 3 == c ? 1.f : 0.f);
      }
    }
  }
  if (lane == 0) {
    stot[warp][0] = wzz;
    stot[warp][1] = wsq;
  }
  __syncthreads();
  double* out = ws + (size_t)blockIdx.x * (E + 2);
  for (int j = threadIdx.x; j < E; j += blockDim.x) {
    double s = 0.0;
    for (int w = 0; w < VQ_WARPS; ++w) s += sz[w][j];
    out[j] = s;
  }
  if (threadIdx.x == 0) {
    double a = 0.0, b = 0.0;
    for (int w = 0; w < VQ_WARPS; ++w) {
      a += stot[w][0];
      b += stot[w][1];
    }
    out[E] = a;
    out[E + 1] = b;
  }
}

// fixed-order tree sum over the block (every thread passes its value; the result is returned to all)
__device__ double block_sum_d(double v, double* red) {
  red[threadIdx.x] = v;
  __syncthreads();
  for (int s = VQ_FIN_THREADS / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  const double r = red[0];
  __syncthreads();
  return r;
}

__global__ void __launch_bounds__(VQ_FIN_THREADS)
vq_finish_kernel(int T, int E, const float* __restrict__ cb, int K, const int* __restrict__ hist,
                 const double* __restrict__ ws, int nblk, float beta, float* __restrict__ scalars) {
  __shared__ double pe[VQ_FIN_THREADS], pee[VQ_FIN_THREADS], red[VQ_FIN_THREADS];
  const int tid = threadIdx.x;
  const int G = VQ_FIN_THREADS / E;                          // groups of E threads, each summing every G-th code
  if (tid < G * E) {
    const int j = tid % E, g = tid / E;
    double s = 0.0, s2 = 0.0;
    for (int k = g; k < K; k += G) {
      const double e = cb[(size_t)k * E + j];
      s += e;
      s2 += e * e;
    }
    pe[tid] = s;
    pee[tid] = s2;
  }
  __syncthreads();
  double dot = 0.0, ee = 0.0;
  for (int j = tid; j < E; j += VQ_FIN_THREADS) {
    double se = 0.0, sz = 0.0;
    for (int g = 0; g < G; ++g) {
      se += pe[g * E + j];
      ee += pee[g * E + j];
    }
    for (int b = 0; b < nblk; ++b) sz += ws[(size_t)b * (E + 2) + j];
    dot += sz * se;
  }
  double ent = 0.0;
  for (int k = tid; k < K; k += VQ_FIN_THREADS) {
    const double pk = (double)hist[k] / T;
    if (pk > 0.0) ent += pk * log(pk + 1e-10);
  }
  dot = block_sum_d(dot, red);
  ee = block_sum_d(ee, red);
  ent = block_sum_d(ent, red);
  if (tid == 0) {
    double zz = 0.0, sq = 0.0;
    for (int b = 0; b < nblk; ++b) {
      zz += ws[(size_t)b * (E + 2) + E];
      sq += ws[(size_t)b * (E + 2) + E + 1];
    }
    const double m = sq / ((double)T * E);
    scalars[0] = (float)(m + (double)beta * m);
    scalars[1] = (float)exp(-ent);
    scalars[2] = (float)(((double)K * zz + (double)T * ee - 2.0 * dot) / ((double)T * K));
  }
}

}  // namespace pgt

using namespace pgt;

extern "C" long long pgt_vq_stats_ws_doubles(int T, int E) {
  return T > 0 && E > 0 ? (long long)vq_grid(T) * (E + 2) : 0;
}

extern "C" int pgt_vq_stats(const float* z, int T, int E, int HW, const float* codebook, int K, const int64_t* idx,
                            float beta, float* zq_nchw, void* zq_bf16, float* min_enc, float* scores, int* usage,
                            int* hist, double* ws, float* scalars, void* stream) {
  PGT_CHECK_ARG(z && codebook && idx && hist && ws && scalars && T > 0 && K > 0 && HW > 0 && T % HW == 0);
  PGT_CHECK_ARG(E > 0 && E % 32 == 0 && E <= VQ_MAX_E && K % 4 == 0);
  PGT_CHECK_ARG(min_enc == nullptr || (reinterpret_cast<uintptr_t>(min_enc) & 15) == 0);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int grid = vq_grid(T);
  {
    const double bytes = (double)T * E * (4 + 4 + (zq_nchw ? 4 : 0) + (zq_bf16 ? 2 : 0)) + (min_enc ? (double)T * K * 4 : 0.0);
    ProfScope ps(PGT_PROF_ARGMAX, bytes, st, "vq_stats");
    vq_token_kernel<<<grid, VQ_WARPS * 32, 0, st>>>(z, T, E, HW, codebook, K, idx, zq_nchw,
                                                   reinterpret_cast<__nv_bfloat16*>(zq_bf16), min_enc, scores, usage,
                                                   hist, ws);
    PGT_LAUNCH_OK();
  }
  {
    ProfScope ps(PGT_PROF_ARGMAX, (double)K * E * 4, st, "vq_finish");
    vq_finish_kernel<<<1, VQ_FIN_THREADS, 0, st>>>(T, E, codebook, K, hist, ws, grid, beta, scalars);
    PGT_LAUNCH_OK();
  }
  return PGT_OK;
}
