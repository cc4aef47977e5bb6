// Residual quantisation over D code levels (RQBottleneck.quantize / embed_code / embed_partial_code /
// embed_code_with_depth, archs/tdcrqvae3_arch.py:294-426).  Each level's nearest code is the exact l2_argmin_tc of the
// level's residual; these two kernels do the elementwise rest:
//   rq_residual_kernel: one quantiser step, e = codebook_d[idx[t]], r_out = r_in - e, agg = agg + e — the reference's
//     residual_feature.sub_(quant) / aggregated_quants.add_(quant) in fp32 (one rounding each, no FMA), so residuals and
//     aggregates are bit-identical to the reference's whenever the codes agree.
//   rq_embed_kernel: out[t] = sum over d in [d0, d1] of codebooks[d][idx[t, d]], accumulated in depth order in fp32
//     (the cat(...).sum(-2) of embed_code, the 'add' / 'select' modes, and PGTFormer's quant_feat).
// r_in may alias r_out (the residual is updated in place after the first depth), so neither is __restrict__.
// Both are memory-bound: one thread per 4 consecutive features of a row.  Indices are not range-checked here; the
// callers check user codes on the host, and argmin / argmax indices are in range by construction.
#include "common.cuh"

namespace pgt {

__global__ void __launch_bounds__(256)
rq_residual_kernel(const float* r_in, float* r_out, const int64_t* __restrict__ idx, int T,
                   int E, const float* __restrict__ cb, float* __restrict__ agg, int first) {
  const int E4 = E >> 2;
  const long long n = (long long)T * E4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int t = (int)(i / E4), j = (int)(i % E4);
    const float4 e = __ldg(reinterpret_cast<const float4*>(cb + idx[t] * E) + j);
    const size_t o = (size_t)t * E4 + j;
    if (r_out != nullptr) {
      const float4 r = reinterpret_cast<const float4*>(r_in)[o];
      reinterpret_cast<float4*>(r_out)[o] =
          make_float4(__fsub_rn(r.x, e.x), __fsub_rn(r.y, e.y), __fsub_rn(r.z, e.z), __fsub_rn(r.w, e.w));
    }
    if (agg == nullptr) continue;
    float4* a = reinterpret_cast<float4*>(agg) + o;
    if (first) {
      *a = e;
    } else {
      const float4 s = *a;
      *a = make_float4(__fadd_rn(s.x, e.x), __fadd_rn(s.y, e.y), __fadd_rn(s.z, e.z), __fadd_rn(s.w, e.w));
    }
  }
}

__global__ void __launch_bounds__(256)
rq_embed_kernel(const int64_t* __restrict__ idx, long long ldi, long long ldd, int T, int d0, int d1,
                const float* __restrict__ cbs, long long cb_stride, int E, void* __restrict__ out, int ldo, int out_dtype) {
  const int E4 = E >> 2;
  const long long n = (long long)T * E4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int t = (int)(i / E4), j = (int)(i % E4);
    const int64_t* it = idx + t * ldi;
    float4 s = __ldg(reinterpret_cast<const float4*>(cbs + d0 * cb_stride + it[d0 * ldd] * E) + j);
    for (int d = d0 + 1; d <= d1; ++d) {
      const float4 e = __ldg(reinterpret_cast<const float4*>(cbs + d * cb_stride + it[d * ldd] * E) + j);
      s = make_float4(__fadd_rn(s.x, e.x), __fadd_rn(s.y, e.y), __fadd_rn(s.z, e.z), __fadd_rn(s.w, e.w));
    }
    if (out_dtype == PGT_BF16) {
      uint2 u;
      u.x = pack_bf16x2(s.x, s.y);
      u.y = pack_bf16x2(s.z, s.w);
      *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(out) + (size_t)t * ldo + 4 * j) = u;
    } else {
      *reinterpret_cast<float4*>(reinterpret_cast<float*>(out) + (size_t)t * ldo + 4 * j) = s;
    }
  }
}

static int elementwise_grid(int T, int E) {
  const long long n = (long long)T * (E >> 2);
  return (int)((n + 255) / 256 < 32LL * num_sms() ? (n + 255) / 256 : 32LL * num_sms());
}

}  // namespace pgt

using namespace pgt;

extern "C" int pgt_rq_residual(const float* r_in, float* r_out, const int64_t* idx, int T, int E, const float* codebook,
                               float* agg, int first, void* stream) {
  PGT_CHECK_ARG(idx && codebook && (agg || r_out) && T > 0 && E > 0 && E % 4 == 0 && (r_out == nullptr || r_in != nullptr));
  PGT_CHECK_ARG(((reinterpret_cast<uintptr_t>(r_in) | reinterpret_cast<uintptr_t>(r_out) |
                  reinterpret_cast<uintptr_t>(codebook) | reinterpret_cast<uintptr_t>(agg)) & 15) == 0);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ProfScope ps(PGT_PROF_ARGMAX, (double)T * E * 4 * (1 + (r_out ? 2 : 0) + (agg ? 2 : 0)) + (double)T * 8, st, "rq_residual");
  rq_residual_kernel<<<elementwise_grid(T, E), 256, 0, st>>>(r_in, r_out, idx, T, E, codebook, agg, first);
  PGT_LAUNCH_OK();
  return PGT_OK;
}

extern "C" int pgt_rq_embed(const int64_t* idx, long long ldi, long long ldd, int T, int d0, int d1,
                            const float* codebooks, long long cb_stride, int E, void* out, int ldo, int out_dtype,
                            void* stream) {
  PGT_CHECK_ARG(idx && codebooks && out && T > 0 && E > 0 && E % 4 == 0 && ldo >= E && ldo % 4 == 0);
  PGT_CHECK_ARG(d0 >= 0 && d1 >= d0 && ldi >= 0 && ldd >= 0 && cb_stride >= 0 && cb_stride % 4 == 0);
  PGT_CHECK_ARG(out_dtype == PGT_F32 || out_dtype == PGT_BF16);
  PGT_CHECK_ARG(((reinterpret_cast<uintptr_t>(codebooks) | reinterpret_cast<uintptr_t>(out)) & 15) == 0);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ProfScope ps(PGT_PROF_ARGMAX, (double)T * E * (4.0 * (d1 - d0 + 1) + (out_dtype == PGT_BF16 ? 2 : 4)), st, "rq_embed");
  rq_embed_kernel<<<elementwise_grid(T, E), 256, 0, st>>>(idx, ldi, ldd, T, d0, d1, codebooks, cb_stride, E, out, ldo,
                                                          out_dtype);
  PGT_LAUNCH_OK();
  return PGT_OK;
}
