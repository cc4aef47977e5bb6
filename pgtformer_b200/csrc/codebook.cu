// RQ-VAE codebook kernels: row argmax + embedding gather (the path PGTFormer.forward takes) and the exhaustive
// fp64 nearest-codebook L2 argmin (the wgmma kernel of the TDCRQVAE3.forward / get_codes path is in
// l2_argmin_tc.cu; this one serves the tokens it cannot certify and the shapes it does not cover).  Index results are
// exact: argmax is a pure fp32 compare; argmin is an fp64 argmin of ||z-e||^2 with lowest index on ties, which is
// stricter than the reference's own fp32 addmm.  Also the multinomial sampler of the soft codes (soft_codes.cu).
#include <curand_kernel.h>
#include <float.h>

#include "common.cuh"

namespace pgt {

// ------------------------------------------------------------------------------ argmax + gather
// One warp per token row: K fp32 logits streamed with 128-bit loads (lane-interleaved float4), running
// (max, first index), warp-shuffle reduction, then the codebook row is gathered cooperatively.
__global__ void __launch_bounds__(256)
argmax_gather_kernel(const float* __restrict__ logits, int T, int K, const float* __restrict__ codebook, int E,
                     const int64_t* __restrict__ idx_in, int64_t* __restrict__ idx_out, void* __restrict__ quant,
                     int ldq, int quant_dtype) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= T) return;
  int best_i;
  if (idx_in != nullptr) {
    best_i = (int)idx_in[row];
  } else {
    const float4* p = reinterpret_cast<const float4*>(logits + (size_t)row * K);
    float best = -FLT_MAX;
    best_i = 0x7fffffff;
    const int nvec = K >> 2;
    for (int i = lane; i < nvec; i += 32) {
      float4 v;
      asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                   : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p + i));
      const int b = i * 4;
      // strictly-greater keeps the first maximum inside the lane's ascending scan
      if (v.x > best) { best = v.x; best_i = b; }
      if (v.y > best) { best = v.y; best_i = b + 1; }
      if (v.z > best) { best = v.z; best_i = b + 2; }
      if (v.w > best) { best = v.w; best_i = b + 3; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, best_i, o);
      if (ov > best || (ov == best && oi < best_i)) { best = ov; best_i = oi; }
    }
  }
  if (lane == 0 && idx_out != nullptr) idx_out[row] = best_i;
  if (quant != nullptr) {
    const float4* src = reinterpret_cast<const float4*>(codebook + (size_t)best_i * E);
    if (quant_dtype == PGT_BF16) {
      __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(quant) + (size_t)row * ldq;
      for (int i = lane; i < (E >> 2); i += 32) {
        const float4 v = __ldg(src + i);
        uint2 u;
        u.x = pack_bf16x2(v.x, v.y);
        u.y = pack_bf16x2(v.z, v.w);
        *reinterpret_cast<uint2*>(dst + i * 4) = u;
      }
    } else {
      float4* dst = reinterpret_cast<float4*>(reinterpret_cast<float*>(quant) + (size_t)row * ldq);
      for (int i = lane; i < (E >> 2); i += 32) dst[i] = __ldg(src + i);
    }
  }
}

// ------------------------------------------------------------------------------ L2 argmin (exhaustive, fp64)
// Every ||z - e_k||^2 is accumulated directly in fp64 (the differences of fp32 values are exact in fp64), running
// (min, first index) per token: this IS the fp64 argmin the tests adjudicate against, for any scale of z and e
// (an fp32 shortlist is not: with ||z|| >> ||e|| all 1024 distances agree to ~1e-6 relative, below fp32 resolution).
// 64 tokens x 64 codes per tile, 4 x 4 fp64 accumulators per thread, two fp64 instructions per term (~3 ms at
// T = 49152, K = 1024, E = 512 on the 64-lane fp64 pipe).  Runs on all T tokens (list == nullptr) for shapes the
// wgmma kernel does not cover, or on the tokens list[0 .. *count) it could not certify — normally none.
constexpr int AM_TT = 64;      // tokens per CTA
constexpr int AM_TC = 64;      // codes per tile
constexpr int AM_KC = 32;      // feature chunk
constexpr int AM_LD = AM_TT + 4;

struct CandD {
  double v;
  int i;
};

__global__ void __launch_bounds__(256)
l2_argmin_kernel(const float* __restrict__ z, int T, int E, const float* __restrict__ cb, int K,
                 int64_t* __restrict__ idx, float* __restrict__ quant, const int* __restrict__ list,
                 const int* __restrict__ count, int min_count) {
  __shared__ __align__(16) float xs[AM_KC][AM_LD];
  __shared__ __align__(16) float es[AM_KC][AM_LD];
  __shared__ CandD merge[AM_TT][16];
  __shared__ int winner[AM_TT];
  const int tx = threadIdx.x & 15;          // code micro-column
  const int ty = threadIdx.x >> 4;          // token micro-row
  const int n_tok = list != nullptr ? *count : T;
  if (list != nullptr && n_tok <= min_count) return;      // short lists belong to l2_argmin_short_list_kernel
  auto token = [&](int i) { return list != nullptr ? list[i] : i; };
  const int lrow = threadIdx.x >> 2;        // 0..63: token / code row this thread stages
  const int lcol = (threadIdx.x & 3) * 8;   // 8 consecutive features
  for (int t0 = blockIdx.x * AM_TT; t0 < n_tok; t0 += gridDim.x * AM_TT) {
    CandD best[4];
#pragma unroll
    for (int a = 0; a < 4; ++a) { best[a].v = DBL_MAX; best[a].i = 0x7fffffff; }
    for (int c0 = 0; c0 < K; c0 += AM_TC) {
      double acc[4][4];
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b] = 0.0;
      for (int k0 = 0; k0 < E; k0 += AM_KC) {
        {
          const int ti = t0 + lrow;
          float4 a = make_float4(0, 0, 0, 0), b = a;
          if (ti < n_tok) {
            const float4* p = reinterpret_cast<const float4*>(z + (size_t)token(ti) * E + k0 + lcol);
            a = __ldg(p); b = __ldg(p + 1);
          }
          xs[lcol + 0][lrow] = a.x; xs[lcol + 1][lrow] = a.y; xs[lcol + 2][lrow] = a.z; xs[lcol + 3][lrow] = a.w;
          xs[lcol + 4][lrow] = b.x; xs[lcol + 5][lrow] = b.y; xs[lcol + 6][lrow] = b.z; xs[lcol + 7][lrow] = b.w;
          const int c = c0 + lrow;
          a = make_float4(0, 0, 0, 0); b = a;
          if (c < K) {
            const float4* p = reinterpret_cast<const float4*>(cb + (size_t)c * E + k0 + lcol);
            a = __ldg(p); b = __ldg(p + 1);
          }
          es[lcol + 0][lrow] = a.x; es[lcol + 1][lrow] = a.y; es[lcol + 2][lrow] = a.z; es[lcol + 3][lrow] = a.w;
          es[lcol + 4][lrow] = b.x; es[lcol + 5][lrow] = b.y; es[lcol + 6][lrow] = b.z; es[lcol + 7][lrow] = b.w;
        }
        __syncthreads();
#pragma unroll 4
        for (int k = 0; k < AM_KC; ++k) {
          const float4 xv = *reinterpret_cast<const float4*>(&xs[k][ty * 4]);
          const float4 ev = *reinterpret_cast<const float4*>(&es[k][tx * 4]);
          const double xa[4] = {(double)xv.x, (double)xv.y, (double)xv.z, (double)xv.w};
          const double ea[4] = {(double)ev.x, (double)ev.y, (double)ev.z, (double)ev.w};
#pragma unroll
          for (int a = 0; a < 4; ++a)
#pragma unroll
            for (int b = 0; b < 4; ++b) {
              const double d = xa[a] - ea[b];
              acc[a][b] = fma(d, d, acc[a][b]);
            }
        }
        __syncthreads();
      }
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) {
          const int c = c0 + tx * 4 + b;                      // ascending within the thread: strict < keeps the first
          if (c < K && acc[a][b] < best[a].v) { best[a].v = acc[a][b]; best[a].i = c; }
        }
    }
    // merge the 16 per-thread minima of each token: lowest index on equal values
#pragma unroll
    for (int a = 0; a < 4; ++a) merge[ty * 4 + a][tx] = best[a];
    __syncthreads();
    if (threadIdx.x < AM_TT) {
      CandD w = merge[threadIdx.x][0];
      for (int j = 1; j < 16; ++j) {
        const CandD c = merge[threadIdx.x][j];
        if (c.v < w.v || (c.v == w.v && c.i < w.i)) w = c;
      }
      winner[threadIdx.x] = w.i;
      if (t0 + threadIdx.x < n_tok) idx[token(t0 + threadIdx.x)] = w.i;
    }
    __syncthreads();
    if (quant != nullptr) {
      const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
      for (int tt = warp; tt < AM_TT; tt += 8) {
        if (t0 + tt >= n_tok) continue;
        const int t = token(t0 + tt), bi = winner[tt];
        for (int e = lane; e < E; e += 32) quant[(size_t)t * E + e] = cb[(size_t)bi * E + e];
      }
    }
    __syncthreads();
  }
}

// The same fp64 argmin for a SHORT token list (the normal case of the wgmma kernel's leftovers: none, or a handful):
// one warp per token, the codebook streamed from L2, so a few tokens spread over the whole chip instead of queueing on
// one CTA of the tiled kernel.  Does nothing when *count > max_count (the tiled kernel takes over).
__global__ void __launch_bounds__(256)
l2_argmin_short_list_kernel(const float* __restrict__ z, int E, const float* __restrict__ cb, int K,
                            int64_t* __restrict__ idx, float* __restrict__ quant, const int* __restrict__ list,
                            const int* __restrict__ count, int max_count) {
  const int n_tok = *count;
  if (n_tok > max_count) return;
  const int lane = threadIdx.x & 31;
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  for (int i = gw; i < n_tok; i += nw) {
    const int t = list[i];
    double bd = DBL_MAX;
    int bi = 0x7fffffff;
    for (int k = 0; k < K; ++k) {
      double s = 0.0;
      for (int e = lane * 4; e < E; e += 128) {
        const float4 a = __ldg(reinterpret_cast<const float4*>(z + (size_t)t * E + e));
        const float4 b = __ldg(reinterpret_cast<const float4*>(cb + (size_t)k * E + e));
        double d;
        d = (double)a.x - (double)b.x; s = fma(d, d, s);
        d = (double)a.y - (double)b.y; s = fma(d, d, s);
        d = (double)a.z - (double)b.z; s = fma(d, d, s);
        d = (double)a.w - (double)b.w; s = fma(d, d, s);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (s < bd) { bd = s; bi = k; }                          // ascending k: strict < keeps the first minimum
    }
    if (lane == 0) idx[t] = bi;
    if (quant != nullptr)
      for (int e = lane; e < E; e += 32) quant[(size_t)t * E + e] = cb[(size_t)bi * E + e];
  }
}

constexpr int AM_SHORT_LIST = 2048;

// ------------------------------------------------------------------------------ multinomial sampling of soft codes
// torch.multinomial(p, 1) of RQBottleneck.get_soft_codes (archs/tdcrqvae3_arch.py:441-444), one warp per row of K
// probabilities (lane l owns the contiguous slice [l * per, (l + 1) * per)).  u in [0, 1) from Philox (key seed[0],
// subsequence = row, offset seed[1]); the code is the first index whose running sum exceeds u * total.  The lane prefix
// is a serial chain (monotone, and unchanged across a lane whose slice is all zeros), and inside the chosen lane a
// zero-probability code never raises the running sum, so such a code is never returned; when rounding leaves no index
// above the threshold the last code with p > 0 is taken.  A row without any positive entry yields -1.  The seed is read
// on the device: no host synchronisation, and a CUDA graph replays fresh draws when seed is refilled before replay.
__global__ void __launch_bounds__(256)
sample_codes_kernel(const float* __restrict__ p, int T, int K, const int64_t* __restrict__ seed, int64_t* __restrict__ idx,
                    int ldp) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  p += (size_t)row * ldp;                                        // row pitch ldp: here, where ptxas keeps it out of the stack
  const int lane = threadIdx.x & 31;
  if (row >= T) return;
  const int per = (K + 31) / 32;
  const int c0 = min(K, lane * per), c1 = min(K, c0 + per);
  const float* pr = p;
  float tot = 0.f;
  int lastnz = -1;
  for (int c = c0; c < c1; ++c) {
    const float v = __ldg(pr + c);
    tot += v;
    if (v > 0.f) lastnz = c;
  }
  float incl = 0.f;
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const float v = __shfl_sync(0xffffffffu, tot, j);
    if (j <= lane) incl += v;
  }
  float excl = __shfl_up_sync(0xffffffffu, incl, 1);
  if (lane == 0) excl = 0.f;
  const float total = __shfl_sync(0xffffffffu, incl, 31);
  float u = 0.f;
  if (lane == 0) {
    curandStatePhilox4_32_10_t st;
    curand_init((unsigned long long)seed[0], (unsigned long long)row, (unsigned long long)seed[1], &st);
    u = 1.f - curand_uniform(&st);                               // (0, 1] -> [0, 1)
  }
  const float x = __shfl_sync(0xffffffffu, u, 0) * total;
  const unsigned above = __ballot_sync(0xffffffffu, incl > x);
  int code = -1;
  if (above != 0) {
    const int sel = __ffs(above) - 1;
    if (lane == sel) {
      float c = excl;
      for (int k = c0; k < c1; ++k) {
        const float v = __ldg(pr + k);
        c += v;
        if (c > x && v > 0.f) { code = k; break; }
      }
      if (code < 0) code = lastnz;                               // incl > excl: this slice has a positive entry
    }
    code = __shfl_sync(0xffffffffu, code, sel);
  } else {
    const unsigned nz = __ballot_sync(0xffffffffu, lastnz >= 0);
    if (nz != 0) code = __shfl_sync(0xffffffffu, lastnz, 31 - __clz(nz));
  }
  if (lane == 0) idx[row] = code;
}

int l2_argmin_list_launch(const float* z, int T, int E, const float* codebook, int K, int64_t* idx, float* quant,
                          const int* list, const int* count, int grid, cudaStream_t st) {
  if (E % AM_KC != 0 || E % 4 != 0) return PGT_ERR_UNSUPPORTED;
  // two launches that look at *count on the device: short lists one warp per token over the whole chip, long lists
  // (degenerate codebooks) through the tiled kernel; with *count == 0 both return at once
  l2_argmin_short_list_kernel<<<num_sms(), 256, 0, st>>>(z, E, codebook, K, idx, quant, list, count, AM_SHORT_LIST);
  PGT_LAUNCH_OK();
  l2_argmin_kernel<<<grid, 256, 0, st>>>(z, T, E, codebook, K, idx, quant, list, count, AM_SHORT_LIST);
  PGT_LAUNCH_OK();
  return PGT_OK;
}

}  // namespace pgt

using namespace pgt;

extern "C" int pgt_argmax_gather(const float* logits, int T, int K, const float* codebook, int E,
                                 const int64_t* idx_in, int64_t* idx, void* quant, int ldq, int quant_dtype,
                                 void* stream) {
  PGT_CHECK_ARG((logits || idx_in) && T > 0 && K > 0 && K % 4 == 0);
  PGT_CHECK_ARG(quant == nullptr || (codebook != nullptr && E % 4 == 0 && ldq % 4 == 0));
  PGT_CHECK_ARG((reinterpret_cast<uintptr_t>(logits) & 15) == 0);
  const int warps = 8;
  ProfScope ps(PGT_PROF_ARGMAX, (double)T * K * 4 + (double)T * 8 + (quant ? (double)T * E * (quant_dtype == PGT_BF16 ? 2 : 4) : 0.0),
               static_cast<cudaStream_t>(stream));
  argmax_gather_kernel<<<ceil_div(T, warps), warps * 32, 0, static_cast<cudaStream_t>(stream)>>>(
      logits, T, K, codebook, E, idx_in, idx, quant, ldq, quant_dtype);
  PGT_LAUNCH_OK();
  return PGT_OK;
}

extern "C" int pgt_sample_codes(const float* p, int T, int K, int ldp, const int64_t* seed, int64_t* idx,
                                void* stream) {
  PGT_CHECK_ARG(p && seed && idx && T > 0 && K > 0 && ldp >= K);
  ProfScope ps(PGT_PROF_ARGMAX, (double)T * K * 4 + (double)T * 8, static_cast<cudaStream_t>(stream), "sample_codes");
  sample_codes_kernel<<<ceil_div(T, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(p, T, K, seed, idx, ldp);
  PGT_LAUNCH_OK();
  return PGT_OK;
}

extern "C" int pgt_l2_argmin(const float* z, int T, int E, const float* codebook, int K, int64_t* idx, float* quant,
                             void* stream) {
  PGT_CHECK_ARG(z && codebook && idx && T > 0 && K > 0 && E > 0 && E % AM_KC == 0);
  PGT_CHECK_ARG((reinterpret_cast<uintptr_t>(z) & 15) == 0 && (reinterpret_cast<uintptr_t>(codebook) & 15) == 0);
  ProfScope ps(PGT_PROF_ARGMIN, 2.0 * T * (double)K * E, static_cast<cudaStream_t>(stream));
  l2_argmin_kernel<<<ceil_div(T, AM_TT), 256, 0, static_cast<cudaStream_t>(stream)>>>(z, T, E, codebook, K, idx, quant, nullptr, nullptr, 0);
  PGT_LAUNCH_OK();
  return PGT_OK;
}
