// Device helpers shared by the wgmma kernels' epilogues.
#pragma once
#include "common.cuh"

namespace pgt {

// Per-(quad, group) partial sums of one 32-column chunk for the fused GroupNorm statistics: each thread reduces
// its row's channels per group (2G values: sum, sumsq), then the warp runs a reduce-scatter butterfly over its 32
// rows — at every step a lane keeps one half of its values and ships the other half to its partner — so the whole
// reduction costs ~2G shuffles instead of 10G; lane (or lane pair ..) i ends up owning value i.
template <int CPG>
__device__ __forceinline__ void gn_chunk_stats(const float (&f)[32], float* gq /*[32 groups][2] of this quad*/, int g0,
                                               int lane) {
  constexpr int G = 32 / CPG;
  constexpr int NV = 2 * G;                    // interleaved (sum, sumsq) per group: value index = g*2 + which
  float v[NV];
#pragma unroll
  for (int g = 0; g < G; ++g) {
    float s = 0.f, q = 0.f;
#pragma unroll
    for (int e = 0; e < CPG; ++e) { const float x = f[g * CPG + e]; s += x; q = fmaf(x, x, q); }
    v[2 * g] = s; v[2 * g + 1] = q;
  }
  int n = NV;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    if (n > 1) {
      const int hlf = n >> 1;
      const bool upper = (lane & o) != 0;
#pragma unroll
      for (int i = 0; i < NV / 2; ++i) {
        if (i < hlf) {
          const float keep = upper ? v[i + hlf] : v[i];
          const float send = upper ? v[i] : v[i + hlf];
          v[i] = keep + __shfl_xor_sync(0xffffffffu, send, o);
        }
      }
      n = hlf;
    } else {
      v[0] += __shfl_xor_sync(0xffffffffu, v[0], o);
    }
  }
  // value index owned by this lane: the lane bits consumed by the splitting steps (offsets 16, 8, ..)
  constexpr int SPLIT = (NV >= 32) ? 5 : (NV >= 16) ? 4 : (NV >= 8) ? 3 : (NV >= 4) ? 2 : 1;
  const int idx = lane >> (5 - SPLIT);
  if ((lane & ((1 << (5 - SPLIT)) - 1)) == 0) gq[g0 * 2 + idx] = v[0];
}


// dispatch on the runtime channels-per-group (N / 32)
__device__ __forceinline__ void gn_chunk_stats_dyn(const float (&f)[32], float* gq, int cpg, int lane) {
  switch (cpg) {
    case 2: gn_chunk_stats<2>(f, gq, 0, lane); break;
    case 4: gn_chunk_stats<4>(f, gq, 0, lane); break;
    case 8: gn_chunk_stats<8>(f, gq, 0, lane); break;
    case 16: gn_chunk_stats<16>(f, gq, 0, lane); break;
    default: gn_chunk_stats<32>(f, gq, 0, lane); break;
  }
}

}  // namespace pgt
