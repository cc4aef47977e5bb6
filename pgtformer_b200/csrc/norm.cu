// GroupNorm(32)+SiLU, LayerNorm and AdaIN on channels-last bf16 activations (HBM-bound kernels:
// 128-bit vector loads, fp32 statistics, deterministic two-level reductions — no atomics).
#include "common.cuh"

namespace pgt {

constexpr int GN_GROUPS = 32;
constexpr int GN_MAX_CHUNKS = 64;
constexpr int GN_THREADS = 512;

__device__ __forceinline__ void load8_bf16(const __nv_bfloat16* p, float (&v)[8]) {
  const uint4 u = __ldg(reinterpret_cast<const uint4*>(p));
  float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
}
__device__ __forceinline__ void store8_bf16(__nv_bfloat16* p, const float (&v)[8]) {
  uint4 u;
  u.x = pack_bf16x2(v[0], v[1]); u.y = pack_bf16x2(v[2], v[3]);
  u.z = pack_bf16x2(v[4], v[5]); u.w = pack_bf16x2(v[6], v[7]);
  *reinterpret_cast<uint4*>(p) = u;
}

// ---------------------------------------------------------------------------------- GroupNorm
// Pass 1: per (frame, pixel-chunk) partial (sum, sumsq) of every group.  Thread (prow, vcol) owns 8 fixed
// channels and strides over the chunk's pixels with 4 independent 16-byte loads in flight; the per-thread sums
// are folded over prow through shared memory in a fixed order (deterministic), then channels -> groups.
__global__ void __launch_bounds__(GN_THREADS)
gn_stats_kernel(const __nv_bfloat16* __restrict__ x, int ldx, int HW, int C, int pix_per_chunk,
                float* __restrict__ partial /*[F][chunks][32][2]*/) {
  extern __shared__ float sm[];              // [rows_par][2][C] per-thread sums, reduced in place
  const int vc = C >> 3;
  const int rows_par = GN_THREADS / vc;
  const int vcol = threadIdx.x % vc;
  const int prow = threadIdx.x / vc;
  const int chunk = blockIdx.x, f = blockIdx.y, nchunks = gridDim.x;
  const int p0 = chunk * pix_per_chunk;
  const int p1 = min(HW, p0 + pix_per_chunk);
  float s[8], q[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { s[i] = 0.f; q[i] = 0.f; }
  if (prow < rows_par) {
    const __nv_bfloat16* base = x + ((size_t)f * HW) * ldx + vcol * 8;
    int p = p0 + prow;
    for (; p + 3 * rows_par < p1; p += 4 * rows_par) {
      float v0[8], v1[8], v2[8], v3[8];
      load8_bf16(base + (size_t)p * ldx, v0);
      load8_bf16(base + (size_t)(p + rows_par) * ldx, v1);
      load8_bf16(base + (size_t)(p + 2 * rows_par) * ldx, v2);
      load8_bf16(base + (size_t)(p + 3 * rows_par) * ldx, v3);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        s[i] += (v0[i] + v1[i]) + (v2[i] + v3[i]);
        q[i] += (v0[i] * v0[i] + v1[i] * v1[i]) + (v2[i] * v2[i] + v3[i] * v3[i]);
      }
    }
    for (; p < p1; p += rows_par) {
      float v[8];
      load8_bf16(base + (size_t)p * ldx, v);
#pragma unroll
      for (int i = 0; i < 8; ++i) { s[i] += v[i]; q[i] += v[i] * v[i]; }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      sm[(prow * 2 + 0) * C + vcol * 8 + i] = s[i];
      sm[(prow * 2 + 1) * C + vcol * 8 + i] = q[i];
    }
  }
  __syncthreads();
  // channel totals: thread c sums its column over prow in a fixed order
  for (int c = threadIdx.x; c < 2 * C; c += GN_THREADS) {
    const int which = c / C, ch = c % C;
    float t = 0.f;
    for (int rr = 0; rr < rows_par; ++rr) t += sm[(rr * 2 + which) * C + ch];
    sm[(size_t)rows_par * 2 * C + c] = t;
  }
  __syncthreads();
  if (threadIdx.x < GN_GROUPS) {
    const float* tot = sm + (size_t)rows_par * 2 * C;
    const int cpg = C / GN_GROUPS;
    float gs = 0.f, gq = 0.f;
    for (int c = threadIdx.x * cpg; c < (threadIdx.x + 1) * cpg; ++c) { gs += tot[c]; gq += tot[C + c]; }
    float* o = partial + (((size_t)f * nchunks + chunk) * GN_GROUPS + threadIdx.x) * 2;
    o[0] = gs; o[1] = gq;
  }
}

// Pass 2 (tiny): fold the chunk partials (fp64) into per-(frame, channel) affine terms
// a = rstd*gamma, b = beta - mean*rstd*gamma, stored after the partials in the workspace.
constexpr int GN_FIN_PARTS = 32;
__global__ void __launch_bounds__(GN_FIN_PARTS * 32)
gn_finalize_kernel(const float* __restrict__ partial, int nchunks, int HW, int C, const float* __restrict__ gamma,
                   const float* __restrict__ beta, float eps, float* __restrict__ ab /*[F][2][C]*/) {
  __shared__ float smean[GN_GROUPS], srstd[GN_GROUPS];
  __shared__ double ps[GN_FIN_PARTS][GN_GROUPS], pq[GN_FIN_PARTS][GN_GROUPS];
  const int f = blockIdx.x;
  const int cpg = C / GN_GROUPS;
  {
    // 32 threads per group stride over the chunks (fused-epilogue statistics come as thousands of per-tile rows;
    // 4 independent loads in flight), then a fixed-order combine: deterministic
    const int g = threadIdx.x & 31, part = threadIdx.x >> 5;
    const float2* base = reinterpret_cast<const float2*>(partial) + (size_t)f * nchunks * GN_GROUPS + g;
    double s = 0.0, q = 0.0;
    int ch = part;
    for (; ch + 3 * GN_FIN_PARTS < nchunks; ch += 4 * GN_FIN_PARTS) {
      const float2 o0 = __ldg(base + (size_t)ch * GN_GROUPS);
      const float2 o1 = __ldg(base + (size_t)(ch + GN_FIN_PARTS) * GN_GROUPS);
      const float2 o2 = __ldg(base + (size_t)(ch + 2 * GN_FIN_PARTS) * GN_GROUPS);
      const float2 o3 = __ldg(base + (size_t)(ch + 3 * GN_FIN_PARTS) * GN_GROUPS);
      s += ((double)o0.x + (double)o1.x) + ((double)o2.x + (double)o3.x);
      q += ((double)o0.y + (double)o1.y) + ((double)o2.y + (double)o3.y);
    }
    for (; ch < nchunks; ch += GN_FIN_PARTS) {
      const float2 o = __ldg(base + (size_t)ch * GN_GROUPS);
      s += (double)o.x; q += (double)o.y;
    }
    ps[part][g] = s; pq[part][g] = q;
  }
  __syncthreads();
  if (threadIdx.x < GN_GROUPS) {
    double s = 0.0, q = 0.0;
    for (int part = 0; part < GN_FIN_PARTS; ++part) { s += ps[part][threadIdx.x]; q += pq[part][threadIdx.x]; }
    const double n = (double)HW * cpg;
    const double mean = s / n;
    double var = q / n - mean * mean;
    if (var < 0.0) var = 0.0;
    smean[threadIdx.x] = (float)mean;
    srstd[threadIdx.x] = (float)(1.0 / sqrt(var + (double)eps));
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const int g = c / cpg;
    const float a = srstd[g] * gamma[c];
    ab[((size_t)f * 2 + 0) * C + c] = a;
    ab[((size_t)f * 2 + 1) * C + c] = beta[c] - smean[g] * a;
  }
}

// Pass 3: y = act(x * a[c] + b[c]); thread (prow, vcol) keeps its 8 channels' a/b in registers and strides over
// pixels with two independent 16-byte loads in flight.
constexpr int GN_APPLY_THREADS = 256;
__global__ void __launch_bounds__(GN_APPLY_THREADS, 3)
gn_apply_kernel(const __nv_bfloat16* __restrict__ x, int ldx, int HW, int C, int pix_per_block,
                const float* __restrict__ ab, int apply_silu, __nv_bfloat16* __restrict__ y, int ldy) {
  const int f = blockIdx.y;
  const int vc = C >> 3;
  const int rows_par = GN_APPLY_THREADS / vc;
  const int vcol = threadIdx.x % vc;
  const int prow = threadIdx.x / vc;
  if (prow >= rows_par) return;
  float a[8], b[8];
  {
    const float4* pa = reinterpret_cast<const float4*>(ab + ((size_t)f * 2 + 0) * C + vcol * 8);
    const float4* pb = reinterpret_cast<const float4*>(ab + ((size_t)f * 2 + 1) * C + vcol * 8);
    const float4 a0 = __ldg(pa), a1 = __ldg(pa + 1), b0 = __ldg(pb), b1 = __ldg(pb + 1);
    a[0] = a0.x; a[1] = a0.y; a[2] = a0.z; a[3] = a0.w; a[4] = a1.x; a[5] = a1.y; a[6] = a1.z; a[7] = a1.w;
    b[0] = b0.x; b[1] = b0.y; b[2] = b0.z; b[3] = b0.w; b[4] = b1.x; b[5] = b1.y; b[6] = b1.z; b[7] = b1.w;
  }
  const int p0 = blockIdx.x * pix_per_block;
  const int p1 = min(HW, p0 + pix_per_block);
  const __nv_bfloat16* xb = x + ((size_t)f * HW) * ldx + vcol * 8;
  __nv_bfloat16* yb = y + ((size_t)f * HW) * ldy + vcol * 8;
  // silu(t) = t*sigmoid(t) = h + h*tanh(h), h = t/2: one MUFU.TANH instead of ex2 + rcp (abs err ~5e-4 of a
  // bf16-rounded result); the 0.5 is folded into the affine terms
  if (apply_silu) {
#pragma unroll
    for (int j = 0; j < 8; ++j) { a[j] *= 0.5f; b[j] *= 0.5f; }
  }
  auto act = [&](float (&v)[8]) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float h = fmaf(v[j], a[j], b[j]);
      float th;
      asm("tanh.approx.f32 %0, %1;" : "=f"(th) : "f"(h));
      v[j] = apply_silu ? fmaf(h, th, h) : h;
    }
  };
  int p = p0 + prow;
  for (; p + 3 * rows_par < p1; p += 4 * rows_par) {       // four independent 16-byte loads in flight per thread
    float v0[8], v1[8], v2[8], v3[8];
    load8_bf16(xb + (size_t)p * ldx, v0);
    load8_bf16(xb + (size_t)(p + rows_par) * ldx, v1);
    load8_bf16(xb + (size_t)(p + 2 * rows_par) * ldx, v2);
    load8_bf16(xb + (size_t)(p + 3 * rows_par) * ldx, v3);
    act(v0); act(v1); act(v2); act(v3);
    store8_bf16(yb + (size_t)p * ldy, v0);
    store8_bf16(yb + (size_t)(p + rows_par) * ldy, v1);
    store8_bf16(yb + (size_t)(p + 2 * rows_par) * ldy, v2);
    store8_bf16(yb + (size_t)(p + 3 * rows_par) * ldy, v3);
  }
  for (; p < p1; p += rows_par) {
    float v[8];
    load8_bf16(xb + (size_t)p * ldx, v);
    act(v);
    store8_bf16(yb + (size_t)p * ldy, v);
  }
}

// ---------------------------------------------------------------------------------- LayerNorm
// One warp per token row, LN_ROWS rows per warp in flight (all loads issued before any reduction) so that
// enough 16-byte requests are outstanding to approach HBM bandwidth; two-pass statistics in registers.
constexpr int LN_ROWS = 4;
// The minimum blocks per SM hold the register budget of the one-pass statistics (the rarely taken shifted pass below
// would otherwise raise it and halve the occupancy of C = 512, the global transformer's width).
template <int NV, bool POS>   // 8-element vectors per lane: C == 256 * NV; POS: second output LN(x) + pos
__global__ void __launch_bounds__(256, NV == 1 ? (POS ? 2 : 3) : (NV == 2 ? 2 : 1))
layernorm_kernel(const void* __restrict__ xin, int ldx, int x_dtype, int T, const float* __restrict__ gamma,
                 const float* __restrict__ beta, float eps, __nv_bfloat16* __restrict__ y, int ldy,
                 const __nv_bfloat16* __restrict__ pos, int ldpos, __nv_bfloat16* __restrict__ y2, int ldy2) {
  constexpr int C = 256 * NV;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int row0 = warp * LN_ROWS;
  if (row0 >= T) return;
  float v[LN_ROWS][NV][8];
  float x0[LN_ROWS];                  // each row's first element: the shift of a row whose one-pass variance cancels
#pragma unroll
  for (int r = 0; r < LN_ROWS; ++r) {
    const int row = min(row0 + r, T - 1);
    x0[r] = x_dtype == PGT_BF16 ? __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(xin)[(size_t)row * ldx])
                                : __ldg(reinterpret_cast<const float*>(xin) + (size_t)row * ldx);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c0 = (i * 32 + lane) * 8;
      if (x_dtype == PGT_BF16) {
        load8_bf16(reinterpret_cast<const __nv_bfloat16*>(xin) + (size_t)row * ldx + c0, v[r][i]);
      } else {
        const float4* p = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(xin) + (size_t)row * ldx + c0);
        const float4 a = __ldg(p), b = __ldg(p + 1);
        v[r][i][0] = a.x; v[r][i][1] = a.y; v[r][i][2] = a.z; v[r][i][3] = a.w;
        v[r][i][4] = b.x; v[r][i][5] = b.y; v[r][i][6] = b.z; v[r][i][7] = b.w;
      }
    }
  }
  // the positional rows of the second output travel with the x rows (issued before any reduction: loading them per row
  // after the statistics exposed one HBM latency per row — 82 us instead of ~45 for the 49152 x 512 launches)
  uint4 pr[POS ? LN_ROWS : 1][NV];
  if constexpr (POS) {
#pragma unroll
    for (int r = 0; r < LN_ROWS; ++r) {
      const int row = min(row0 + r, T - 1);
#pragma unroll
      for (int i = 0; i < NV; ++i)
        pr[r][i] = __ldg(reinterpret_cast<const uint4*>(pos + (size_t)row * ldpos + (i * 32 + lane) * 8));
    }
  }
  float g[NV][8], bt[NV][8];
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c0 = (i * 32 + lane) * 8;
    const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + c0)), g1 = __ldg(reinterpret_cast<const float4*>(gamma + c0 + 4));
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + c0)), b1 = __ldg(reinterpret_cast<const float4*>(beta + c0 + 4));
    g[i][0] = g0.x; g[i][1] = g0.y; g[i][2] = g0.z; g[i][3] = g0.w; g[i][4] = g1.x; g[i][5] = g1.y; g[i][6] = g1.z; g[i][7] = g1.w;
    bt[i][0] = b0.x; bt[i][1] = b0.y; bt[i][2] = b0.z; bt[i][3] = b0.w; bt[i][4] = b1.x; bt[i][5] = b1.y; bt[i][6] = b1.z; bt[i][7] = b1.w;
  }
  // the kernel is issue-bound before it is HBM-bound (10 instructions per element with two-pass statistics):
  // one pass (sum, sum of squares) and the normalisation as two FMAs per element
#pragma unroll
  for (int r = 0; r < LN_ROWS; ++r) {
    const int row = row0 + r;
    float s = 0.f, q = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) { s += v[r][i][j]; q = fmaf(v[r][i][j], v[r][i][j], q); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      s += __shfl_xor_sync(0xffffffffu, s, o);
      q += __shfl_xor_sync(0xffffffffu, q, o);
    }
    float mean = s * (1.0f / C);
    float var = q * (1.0f / C) - mean * mean;
    // A row far from zero next to its spread (|mean| >= 32 std, or constant; e.g. the global transformer's fp32
    // residual stream) makes q / C - mean^2 cancel: a relative variance error of ~2^-24 (mean / std)^2, and worse from
    // the fp32 sums.  Such a row is summed again, shifted by one of its own elements, and normalised shifted too: a
    // constant row then gives exactly beta.  Every other row keeps the one-pass sums (and its bits).  The butterfly
    // sums are identical on every lane, so the branch is warp-uniform.
    float piv = 0.f;
    if (!(var * 1024.f > mean * mean)) {
      piv = x0[r];
      s = 0.f;
      q = 0.f;
#pragma unroll
      for (int i = 0; i < NV; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float d = v[r][i][j] - piv;
          s += d;
          q = fmaf(d, d, q);
        }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        s += __shfl_xor_sync(0xffffffffu, s, o);
        q += __shfl_xor_sync(0xffffffffu, q, o);
      }
      mean = s * (1.0f / C);
      var = q * (1.0f / C) - mean * mean;
    }
    const float rstd = rsqrtf(fmaxf(var, 0.f) + eps);
    const float nm = -mean * rstd;
    if (row < T) {
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int c0 = (i * 32 + lane) * 8;
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = fmaf(fmaf(v[r][i][j] - piv, rstd, nm), g[i][j], bt[i][j]);
        store8_bf16(y + (size_t)row * ldy + c0, o);
        if constexpr (POS) {
          const uint32_t pw[4] = {pr[r][i].x, pr[r][i].y, pr[r][i].z, pr[r][i].w};
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float2 pv = unpack_bf16x2(pw[j]);
            o[2 * j] += pv.x; o[2 * j + 1] += pv.y;
          }
          store8_bf16(y2 + (size_t)row * ldy2 + c0, o);
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------- AdaIN
// Block = (frame, 64-channel slab).  Thread (prow, vcol) strides over pixels accumulating fp32 (sum, sumsq)
// for content q and style l; block reduce; second sweep applies the affine map.  kFlags (pgt_adain_frames): a frame
// whose flag is 0 is only rounded to bf16.
constexpr int ADAIN_THREADS = 256;
template <bool kFlags>
__global__ void __launch_bounds__(ADAIN_THREADS)
adain_kernel(const void* __restrict__ qin, int ldq, int q_dtype, const __nv_bfloat16* __restrict__ l, int ldl, int HW,
             int C, float eps, const int* __restrict__ flags, __nv_bfloat16* __restrict__ y, int ldy) {
  __shared__ float red[4][ADAIN_THREADS / 8][64];   // [stat][prow][channel]
  __shared__ float sa[64], sb[64], spiv[64];
  __shared__ double sml[64], ssl[64];
  const int f = blockIdx.y;
  const int cbase = blockIdx.x * 64;
  const int vcol = threadIdx.x & 7;
  const int prow = threadIdx.x >> 3;
  const int rows_par = ADAIN_THREADS / 8;
  const int c0 = cbase + vcol * 8;
  auto load_q = [&](int p, float (&v)[8]) {
    if (q_dtype == PGT_BF16) {
      load8_bf16(reinterpret_cast<const __nv_bfloat16*>(qin) + ((size_t)f * HW + p) * ldq + c0, v);
    } else {
      const float4* pp = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(qin) + ((size_t)f * HW + p) * ldq + c0);
      const float4 a = __ldg(pp), b = __ldg(pp + 1);
      v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    }
  };
  if constexpr (kFlags) {
    if (flags[f] == 0) {                                // uniform over the block
      for (int p = prow; p < HW; p += rows_par) {
        float vq[8];
        load_q(p, vq);
        store8_bf16(y + ((size_t)f * HW + p) * ldy + c0, vq);
      }
      return;
    }
  }
  float acc[4][8];
#pragma unroll
  for (int k = 0; k < 4; ++k)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[k][j] = 0.f;
  for (int p = prow; p < HW; p += rows_par) {
    float vq[8], vl[8];
    load_q(p, vq);
    load8_bf16(l + ((size_t)f * HW + p) * ldl + c0, vl);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      acc[0][j] += vq[j]; acc[1][j] += vq[j] * vq[j];
      acc[2][j] += vl[j]; acc[3][j] += vl[j] * vl[j];
    }
  }
#pragma unroll
  for (int k = 0; k < 4; ++k)
#pragma unroll
    for (int j = 0; j < 8; ++j) red[k][prow][vcol * 8 + j] = acc[k][j];
  __syncthreads();
  bool shift = false;
  if (threadIdx.x < 64) {
    double s[4] = {0, 0, 0, 0};
    for (int r = 0; r < rows_par; ++r)
#pragma unroll
      for (int k = 0; k < 4; ++k) s[k] += (double)red[k][r][threadIdx.x];
    const double n = (double)HW;
    const double mq = s[0] / n, ml = s[2] / n;
    double vq = (s[1] - n * mq * mq) / (n - 1.0), vl = (s[3] - n * ml * ml) / (n - 1.0);   // unbiased (torch.var)
    // a content channel far from zero next to its spread (|mean| >= 32 std, or constant): its fp32 sums of squares
    // cancel against n * mean^2, so it is summed again below, shifted by its value at pixel 0
    shift = !(vq * 1024.0 > mq * mq);
    if (vq < 0) vq = 0;
    if (vl < 0) vl = 0;
    const double sq = sqrt(vq + (double)eps), sl = sqrt(vl + (double)eps);
    const double a = sl / sq;
    sa[threadIdx.x] = (float)a;
    sb[threadIdx.x] = (float)(ml - mq * a);
    sml[threadIdx.x] = ml;
    ssl[threadIdx.x] = sl;
    float piv = 0.f;
    if (shift) {
      const size_t i0 = (size_t)f * HW * ldq + cbase + threadIdx.x;
      piv = q_dtype == PGT_BF16 ? __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(qin)[i0])
                                : reinterpret_cast<const float*>(qin)[i0];
    }
    spiv[threadIdx.x] = piv;                            // 0 for every other channel: their bits are unchanged
  }
  if (__syncthreads_or(shift)) {                        // rare: a second pass over the content of this slab
    float pq[8], a2[2][8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { pq[j] = spiv[vcol * 8 + j]; a2[0][j] = 0.f; a2[1][j] = 0.f; }
    for (int p = prow; p < HW; p += rows_par) {
      float vq[8];
      load_q(p, vq);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = vq[j] - pq[j];
        a2[0][j] += d; a2[1][j] += d * d;
      }
    }
#pragma unroll
    for (int k = 0; k < 2; ++k)
#pragma unroll
      for (int j = 0; j < 8; ++j) red[k][prow][vcol * 8 + j] = a2[k][j];
    __syncthreads();
    if (shift) {
      double s0 = 0, s1 = 0;
      for (int r = 0; r < rows_par; ++r) { s0 += (double)red[0][r][threadIdx.x]; s1 += (double)red[1][r][threadIdx.x]; }
      const double n = (double)HW;
      const double mq = s0 / n;                         // mean of the shifted channel
      double vq = (s1 - n * mq * mq) / (n - 1.0);
      if (vq < 0) vq = 0;
      const double a = ssl[threadIdx.x] / sqrt(vq + (double)eps);
      sa[threadIdx.x] = (float)a;
      sb[threadIdx.x] = (float)(sml[threadIdx.x] - mq * a);   // applied to the shifted content
    }
  }
  __syncthreads();
  for (int p = prow; p < HW; p += rows_par) {
    float vq[8];
    load_q(p, vq);
#pragma unroll
    for (int j = 0; j < 8; ++j) vq[j] = (vq[j] - spiv[vcol * 8 + j]) * sa[vcol * 8 + j] + sb[vcol * 8 + j];
    store8_bf16(y + ((size_t)f * HW + p) * ldy + c0, vq);
  }
}

}  // namespace pgt

using namespace pgt;

static int gn_chunks(int HW) {
  int c = ceil_div(HW, 1024);
  return c < 1 ? 1 : (c > GN_MAX_CHUNKS ? GN_MAX_CHUNKS : c);
}

extern "C" int64_t pgt_groupnorm_ws_floats(int F, int HW, int C) {
  return (int64_t)F * gn_chunks(HW) * GN_GROUPS * 2 + (int64_t)F * 2 * C;
}

extern "C" int pgt_groupnorm_silu(const void* x, int ldx, int F, int HW, int C, const float* gamma, const float* beta,
                                  float eps, int apply_silu, void* y, int ldy, float* ws, void* stream) {
  PGT_CHECK_ARG(x && y && ws && gamma && beta && F > 0 && HW > 0);
  PGT_CHECK_ARG(C % 32 == 0 && C % 8 == 0 && C / 8 <= GN_APPLY_THREADS && ldx % 8 == 0 && ldy % 8 == 0);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ProfScope ps(PGT_PROF_NORM, 3.0 * F * (double)HW * C * 2, st);     // read, read, write (bf16)
  const int nchunks = gn_chunks(HW);
  const int ppc = ceil_div(HW, nchunks);
  float* ab = ws + (size_t)F * nchunks * GN_GROUPS * 2;
  const size_t stats_smem = ((size_t)(GN_THREADS / (C / 8)) + 1) * 2 * C * sizeof(float);   // <= 2*(512*8+C)*4 B
  gn_stats_kernel<<<dim3(nchunks, F), GN_THREADS, stats_smem, st>>>(
      reinterpret_cast<const __nv_bfloat16*>(x), ldx, HW, C, ppc, ws);
  PGT_LAUNCH_OK();
  gn_finalize_kernel<<<F, GN_FIN_PARTS * 32, 0, st>>>(ws, nchunks, HW, C, gamma, beta, eps, ab);
  PGT_LAUNCH_OK();
  // apply: ~128 KB of activations per block
  int ppb = (131072 / (C * 2));
  if (ppb < 16) ppb = 16;
  const int nblk = ceil_div(HW, ppb);
  gn_apply_kernel<<<dim3(nblk, F), GN_APPLY_THREADS, 0, st>>>(
      reinterpret_cast<const __nv_bfloat16*>(x), ldx, HW, C, ppb, ab, apply_silu,
      reinterpret_cast<__nv_bfloat16*>(y), ldy);
  PGT_LAUNCH_OK();
  return PGT_OK;
}

extern "C" int pgt_groupnorm_apply_stats(const void* x, int ldx, int F, int HW, int C, const float* gamma,
                                         const float* beta, float eps, int apply_silu, void* y, int ldy,
                                         const float* stats, int chunks_per_frame, float* ws, void* stream) {
  PGT_CHECK_ARG(x && y && ws && gamma && beta && stats && F > 0 && HW > 0 && chunks_per_frame > 0);
  PGT_CHECK_ARG(C % 32 == 0 && C % 8 == 0 && C / 8 <= GN_APPLY_THREADS && ldx % 8 == 0 && ldy % 8 == 0);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ProfScope ps(PGT_PROF_NORM, 2.0 * F * (double)HW * C * 2, st, "gn_apply_stats");   // read + write (bf16)
  gn_finalize_kernel<<<F, GN_FIN_PARTS * 32, 0, st>>>(stats, chunks_per_frame, HW, C, gamma, beta, eps, ws);
  PGT_LAUNCH_OK();
  int ppb = (131072 / (C * 2));
  if (ppb < 16) ppb = 16;
  gn_apply_kernel<<<dim3(ceil_div(HW, ppb), F), GN_APPLY_THREADS, 0, st>>>(
      reinterpret_cast<const __nv_bfloat16*>(x), ldx, HW, C, ppb, ws, apply_silu, reinterpret_cast<__nv_bfloat16*>(y), ldy);
  PGT_LAUNCH_OK();
  return PGT_OK;
}

// finalize only: per-(frame, channel) affine terms for a consumer that applies the normalisation itself
extern "C" int pgt_groupnorm_ab(const void* x, int ldx, int F, int HW, int C, const float* gamma, const float* beta,
                                float eps, const float* stats, int chunks_per_frame, float* ws, float* ab, void* stream) {
  PGT_CHECK_ARG(gamma && beta && ab && F > 0 && HW > 0 && C % 32 == 0 && C / 8 <= GN_APPLY_THREADS);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (stats != nullptr) {
    PGT_CHECK_ARG(chunks_per_frame > 0);
    gn_finalize_kernel<<<F, GN_FIN_PARTS * 32, 0, st>>>(stats, chunks_per_frame, HW, C, gamma, beta, eps, ab);
    PGT_LAUNCH_OK();
    return PGT_OK;
  }
  PGT_CHECK_ARG(x && ws && ldx % 8 == 0);
  ProfScope ps(PGT_PROF_NORM, 1.0 * F * (double)HW * C * 2, st, "gn_stats");
  const int nchunks = gn_chunks(HW);
  const int ppc = ceil_div(HW, nchunks);
  const size_t stats_smem = ((size_t)(GN_THREADS / (C / 8)) + 1) * 2 * C * sizeof(float);
  gn_stats_kernel<<<dim3(nchunks, F), GN_THREADS, stats_smem, st>>>(reinterpret_cast<const __nv_bfloat16*>(x), ldx, HW, C, ppc, ws);
  PGT_LAUNCH_OK();
  gn_finalize_kernel<<<F, GN_FIN_PARTS * 32, 0, st>>>(ws, nchunks, HW, C, gamma, beta, eps, ab);
  PGT_LAUNCH_OK();
  return PGT_OK;
}

extern "C" int pgt_layernorm(const void* x, int ldx, int x_dtype, int T, int C, const float* gamma, const float* beta,
                             float eps, void* y, int ldy, const void* pos, int ldpos, void* y2, int ldy2,
                             void* stream) {
  PGT_CHECK_ARG(x && y && gamma && beta && T > 0);
  PGT_CHECK_ARG(C % 256 == 0 && C <= 1024 && ldx % 8 == 0 && ldy % 8 == 0);
  PGT_CHECK_ARG(y2 == nullptr || (pos != nullptr && ldpos % 8 == 0 && ldy2 % 8 == 0));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ProfScope ps(7, (double)T * C * ((x_dtype == PGT_BF16 ? 2.0 : 4.0) + 2.0 + (y2 ? 4.0 : 0.0)), st, "layernorm");
  const int warps_per_block = 8;
  const int grid = ceil_div(T, warps_per_block * LN_ROWS);
  auto yb = reinterpret_cast<__nv_bfloat16*>(y);
  auto pb = reinterpret_cast<const __nv_bfloat16*>(pos);
  auto y2b = reinterpret_cast<__nv_bfloat16*>(y2);
#define PGT_LN_LAUNCH(NV_)                                                                                              \
  do {                                                                                                                \
    if (y2b != nullptr) layernorm_kernel<NV_, true><<<grid, 256, 0, st>>>(x, ldx, x_dtype, T, gamma, beta, eps, yb, ldy, pb, ldpos, y2b, ldy2); \
    else layernorm_kernel<NV_, false><<<grid, 256, 0, st>>>(x, ldx, x_dtype, T, gamma, beta, eps, yb, ldy, pb, ldpos, y2b, ldy2);           \
  } while (0)
  if (C == 256) PGT_LN_LAUNCH(1);
  else if (C == 512) PGT_LN_LAUNCH(2);
  else if (C == 768) PGT_LN_LAUNCH(3);
  else PGT_LN_LAUNCH(4);
#undef PGT_LN_LAUNCH
  PGT_LAUNCH_OK();
  return PGT_OK;
}

extern "C" int pgt_adain(const void* q, int ldq, int q_dtype, const void* l, int ldl, int F, int HW, int C, float eps,
                         void* y, int ldy, void* stream) {
  PGT_CHECK_ARG(q && l && y && F > 0 && HW > 1 && C % 64 == 0 && ldq % 8 == 0 && ldl % 8 == 0 && ldy % 8 == 0);
  ProfScope ps(PGT_PROF_MOVE, 8.0 * F * (double)HW * C, static_cast<cudaStream_t>(stream), "adain");
  adain_kernel<false><<<dim3(C / 64, F), ADAIN_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
      q, ldq, q_dtype, reinterpret_cast<const __nv_bfloat16*>(l), ldl, HW, C, eps, nullptr,
      reinterpret_cast<__nv_bfloat16*>(y), ldy);
  PGT_LAUNCH_OK();
  return PGT_OK;
}

extern "C" int pgt_adain_frames(const void* q, int ldq, int q_dtype, const void* l, int ldl, int F, int HW, int C,
                                float eps, const int32_t* flags, void* y, int ldy, void* stream) {
  PGT_CHECK_ARG(q && l && y && flags && F > 0 && HW > 1 && C % 64 == 0 && ldq % 8 == 0 && ldl % 8 == 0 && ldy % 8 == 0);
  ProfScope ps(PGT_PROF_MOVE, 8.0 * F * (double)HW * C, static_cast<cudaStream_t>(stream), "adain_frames");
  adain_kernel<true><<<dim3(C / 64, F), ADAIN_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
      q, ldq, q_dtype, reinterpret_cast<const __nv_bfloat16*>(l), ldl, HW, C, eps, flags,
      reinterpret_cast<__nv_bfloat16*>(y), ldy);
  PGT_LAUNCH_OK();
  return PGT_OK;
}
