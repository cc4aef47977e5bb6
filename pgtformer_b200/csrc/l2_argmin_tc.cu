// Nearest-codebook L2 argmin (VQEmbedding.compute_distances + find_nearest_embedding, archs/tdcrqvae3_arch.py:99-126)
// on wgmma, exact by construction.
//
//   argmin_k ||z - e_k||^2  =  argmin_k ( ||e_k||^2 - 2 z.e_k )        (||z||^2 is constant per token)
//
// Pass 0 (z_pack_kernel, HBM-bound): the fp32 z rows are read ONCE with 128-bit streaming loads and written back as bf16
//   rows z~ together with (||z||^2, ||z - z~||^2) per token (needed for the certificate below).
// Pass 1 (l2_argmin_tc_kernel, tensor cores): the scores  s~ = z~ . e~_k  of the bf16-rounded operands for all K codes,
//   128 tokens per CTA, N-tile = 128 codes, k-block = 64:
//   * the CTA keeps its 128 tokens' A tile (128 x E bf16) resident in shared memory and streams the codebook tiles
//     through a TMA ring; persistent over 128-token tiles, the A k-blocks of the next tile are loaded by their own
//     producer warp (per-k-block barriers) as soon as the last N-tile of the current one has consumed them;
//   * two warpgroups, warpgroup h owning token rows [64h, 64h + 64): wgmma 64 x 128 x 16 into registers, then 32 codes at
//     a time through a shared-memory exchange to two threads per token row (16 codes each): d~_k = ||e_k||^2 - 2 s~,
//     BRANCH-FREE chunk minimum, and ONE test per chunk (chunk min <= running min + W); only then the chunk's codes within
//     W of the (updated) running minimum are appended, with predicated stores, to the thread's candidate list in shared
//     memory.  The list is emptied whenever the minimum drops by more than W, so it is a superset of the final window
//     {k : d~_k <= min d~ + W}.  (A test-and-branch per code costs tens of cycles of dependent latency each.)
//   * merge (all 256 threads: each filters its own list against the row's global minimum) and exact resolution (below).
// Certificate: |d~_k - d_k| <= D := 2 (||z - z~|| max||e~|| + ||z|| max||e - e~||) + slack (Cauchy-Schwarz on the two
//   rounding-error dot products + fp32 accumulation slack), hence the true argmin lies in {k : d~_k <= min d~ + 2D},
//   W = 2D.  The window's members (usually ONE) are re-evaluated exactly — fp32 direct sums, whose relative error is
//   bounded by 23 ulp, decide unless two candidates are closer than that bound, in which case fp64 decides (lowest
//   index on ties).  Rows whose window holds more than 16 codes or whose list overflowed (degenerate codebooks: many
//   duplicated / zero rows) are appended to a list for the exhaustive fp32+fp64 kernel in codebook.cu.
// The result therefore equals an fp64 argmin of ||z - e_k||^2 with first-index tie-break for every input.
//
// Codebook split (pgt_l2_argmin_tc_split, small T): the grid is token tiles x S code ranges of whole 128-code N-tiles
// (the last one ragged).  Each CTA runs the same scan over its range and writes, per (token, range, list owner), its
// running minimum d~, its candidate list and the list length (> LT_LIST: overflow) to the workspace instead of merging.
// l2_argmin_merge_kernel (one warp per token) takes the global minimum, keeps every list's entries within W of it and
// resolves them exactly as above; overflowed lists and windows of more than LT_TOP codes go to the exhaustive kernel.
// Exact for any S: each list is a superset of {k in its range : d~_k <= its range's min + W}, and the global minimum is
// <= every range's minimum, so the lists together hold the whole global window.
#include <float.h>

#include "common.cuh"
#include "ptx.cuh"
#include "tmap.cuh"

namespace pgt {

constexpr int LT_BM = 128;                       // tokens per CTA
constexpr int LT_BN = 128;                       // codes per N-tile
constexpr int LT_BK = 64;                        // k-block (one 128-byte swizzled row)
constexpr int LT_EMAX = 512;                     // A tile resident: 128 x 512 bf16 = 128 KB
constexpr int LT_A_KB_BYTES = LT_BM * 128;       // 16 KB per k-block of A
constexpr int LT_KBMAX = LT_EMAX / LT_BK;        // 8
constexpr int LT_BST = LT_BN * 128;              // codebook stage: 128 codes x 64 k = 16 KB
constexpr int LT_NST = 2;                        // codebook ring depth
constexpr int LT_THREADS = 10 * 32;              // warps: 0..7 MMA / scan / resolve, 8 codebook producer, 9 A producer
constexpr int LT_SCH = 16;                       // codes per thread per exchange round
constexpr int LT_XLD = 36;                       // exchange pitch (fp32): [2 warpgroups][64 rows][32 codes + pad]
constexpr int LT_TOP = 16;                       // window members resolved in-kernel (more -> exhaustive kernel)
constexpr int LT_LIST = 16;                      // candidate-list capacity per (token, warpgroup)
constexpr int LT_XCH = 2 * LT_BM * LT_LIST * 8 /*lists*/ + 2 * LT_BM * 4 /*xmin*/ + LT_BM * LT_TOP * 4 /*mi*/ + 2 * LT_BM * 4 /*ncand, ovf*/;
constexpr int LT_XACC = LT_BM * LT_XLD * 4;
constexpr int LT_SMEM = LT_BM * LT_EMAX * 2 + LT_NST * LT_BST + LT_XCH + LT_XACC + 512 /*barriers*/ + 1024 /*align*/;
static_assert(LT_SMEM <= 232448, "l2_argmin smem budget");

__device__ __forceinline__ float4 ld_nc_f4(const float4* p) {       // streaming 128-bit load (read once, keep out of L1)
  float4 v;
  asm("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
  return v;
}

// ------------------------------------------------------------------------------ codebook pack (load time)
// bf16 copy of the codebook, ||e_k||^2 (fp64 sum rounded to fp32) and the two maxima the certificate needs:
// norm[K] = max_k ||e~_k||, norm[K+1] = max_k ||e_k - e~_k|| (written as squared maxima, finalised by the caller kernel).
__global__ void __launch_bounds__(256)
codebook_pack_kernel(const float* __restrict__ cb, int K, int E, __nv_bfloat16* __restrict__ cb16, float* __restrict__ norm) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= K) return;
  double s = 0.0;
  float sr = 0.f, sd = 0.f;
  for (int e = lane; e < E; e += 32) {
    const float v = cb[(size_t)row * E + e];
    const __nv_bfloat16 b = __float2bfloat16_rn(v);
    const float vb = __bfloat162float(b);
    cb16[(size_t)row * E + e] = b;
    s += (double)v * (double)v;
    sr = fmaf(vb, vb, sr);
    const float dd = v - vb;
    sd = fmaf(dd, dd, sd);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    sr += __shfl_xor_sync(0xffffffffu, sr, o);
    sd += __shfl_xor_sync(0xffffffffu, sd, o);
  }
  if (lane == 0) {
    norm[row] = (float)s;
    // non-negative floats order like their bit patterns
    atomicMax(reinterpret_cast<int*>(norm + K), __float_as_int(sr * 1.0001f));
    atomicMax(reinterpret_cast<int*>(norm + K + 1), __float_as_int(sd * 1.0001f));
  }
}

// ------------------------------------------------------------------------------ z pack (pass 0)
__global__ void __launch_bounds__(256)
z_pack_kernel(const float* __restrict__ z, int T, int E, __nv_bfloat16* __restrict__ zb, float2* __restrict__ zn2) {
  constexpr int RB = 4;
  const int lane = threadIdx.x & 31;
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  const int nstep = (E + 255) / 256;
  for (int t0 = gw * RB; t0 < T; t0 += nw * RB) {
    float4 va[RB][2][2];
#pragma unroll
    for (int i = 0; i < RB; ++i) {
#pragma unroll
      for (int sp = 0; sp < 2; ++sp) {
        const int c = sp * 256 + lane * 8;
        if (sp < nstep && t0 + i < T && c < E) {
          const float4* p = reinterpret_cast<const float4*>(z + (size_t)(t0 + i) * E + c);
          va[i][sp][0] = ld_nc_f4(p);
          va[i][sp][1] = ld_nc_f4(p + 1);
        } else {
          va[i][sp][0] = va[i][sp][1] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
    }
#pragma unroll
    for (int i = 0; i < RB; ++i) {
      const int t = t0 + i;
      if (t >= T) break;
      float s2 = 0.f, d2 = 0.f;
#pragma unroll
      for (int sp = 0; sp < 2; ++sp) {
        const int c = sp * 256 + lane * 8;
        if (sp < nstep && c < E) {
          const float4 a = va[i][sp][0], b = va[i][sp][1];
          const float f[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
          uint32_t u[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            u[q] = pack_bf16x2(f[2 * q], f[2 * q + 1]);
            const float2 back = unpack_bf16x2(u[q]);
            s2 = fmaf(f[2 * q], f[2 * q], s2); s2 = fmaf(f[2 * q + 1], f[2 * q + 1], s2);
            const float e0 = f[2 * q] - back.x, e1 = f[2 * q + 1] - back.y;      // exact in fp32
            d2 = fmaf(e0, e0, d2); d2 = fmaf(e1, e1, d2);
          }
          *reinterpret_cast<uint4*>(zb + (size_t)t * E + c) = make_uint4(u[0], u[1], u[2], u[3]);
        }
      }
      s2 = warp_sum(s2); d2 = warp_sum(d2);
      if (lane == 0) zn2[t] = make_float2(s2, d2);
    }
  }
}

// ------------------------------------------------------------------------------ scan / merge / exact resolution
// Scan of LT_SCH consecutive scores s~ of this thread's token row (see the header comment).  lst_s: the shared-window
// address of this thread's candidate list, entry j 2 * LT_BM entries further (entry-major: the lanes of a warp hit
// distinct banks).
__device__ __forceinline__ void argmin_scan_chunk(const uint32_t (&v)[LT_SCH], const float* __restrict__ norm_c, int cbase,
                                                  float W, uint32_t lst_s, float& runmin, float& thr, int& cnt) {
  uint32_t laddr = lst_s + (uint32_t)cnt * (2 * LT_BM * 8);   // shared-window address of the next list entry
  const float4* np = reinterpret_cast<const float4*>(norm_c);
  float d[LT_SCH];
#pragma unroll
  for (int q = 0; q < LT_SCH / 4; ++q) {
    const float4 n4 = __ldg(np + q);
    d[4 * q] = n4.x; d[4 * q + 1] = n4.y; d[4 * q + 2] = n4.z; d[4 * q + 3] = n4.w;
  }
  float m0 = FLT_MAX, m1 = FLT_MAX, m2 = FLT_MAX, m3 = FLT_MAX;
#pragma unroll
  for (int i = 0; i < LT_SCH; i += 4) {
    d[i] = fmaf(-2.f, __uint_as_float(v[i]), d[i]);             m0 = fminf(m0, d[i]);
    d[i + 1] = fmaf(-2.f, __uint_as_float(v[i + 1]), d[i + 1]); m1 = fminf(m1, d[i + 1]);
    d[i + 2] = fmaf(-2.f, __uint_as_float(v[i + 2]), d[i + 2]); m2 = fminf(m2, d[i + 2]);
    d[i + 3] = fmaf(-2.f, __uint_as_float(v[i + 3]), d[i + 3]); m3 = fminf(m3, d[i + 3]);
  }
  const float cm = fminf(fminf(m0, m1), fminf(m2, m3));
  if (cm <= thr) {                                         // the only branch of the chunk (dead rows: thr = -FLT_MAX)
    if (cm < runmin) {
      if (cm + W < runmin) { cnt = 0; laddr = lst_s; }     // every earlier entry is now outside any final window
      runmin = cm; thr = cm + W;
    }
    // predicated append of every code of the chunk within W of the running minimum — no branch per code
#pragma unroll
    for (int i = 0; i < LT_SCH; ++i) {
      asm volatile(
          "{\n\t.reg .pred h, p;\n\t"
          "setp.le.f32 h, %2, %3;\n\t"
          "setp.lt.and.s32 p, %0, %5, h;\n\t"
          "@p st.shared.v2.b32 [%1], {%6, %4};\n\t"
          "@h add.s32 %0, %0, 1;\n\t"
          "@h add.u32 %1, %1, %7;\n\t}"
          : "+r"(cnt), "+r"(laddr)
          : "f"(d[i]), "f"(thr), "r"(cbase + i), "n"(LT_LIST), "r"(__float_as_uint(d[i])), "n"(2 * LT_BM * 8)
          : "memory");
    }
  }
}

__device__ __forceinline__ void argmin_load_row(const float* __restrict__ p, int E, int lane, float4 (&r)[LT_EMAX / 128]) {
#pragma unroll
  for (int q = 0; q < LT_EMAX / 128; ++q)
    r[q] = (q * 128 + lane * 4 < E) ? __ldg(reinterpret_cast<const float4*>(p) + q * 32 + lane) : make_float4(0.f, 0.f, 0.f, 0.f);
}

// Exact resolution of one token by one warp: the n (> 1) members of its window re-evaluated with fp32 direct sums (the rows
// of up to four candidates are in flight together), fp64 when two of them are closer than the fp32 error bound; lowest
// index on ties.  Returns the code in every lane.
__device__ __forceinline__ int argmin_resolve_exact(const float* __restrict__ z, const float* __restrict__ cb, int E, int t, int n,
                                                    const int* mi_row, int lane) {
  float4 zr[LT_EMAX / 128];
  argmin_load_row(z + (size_t)t * E, E, lane, zr);
  float b1 = FLT_MAX, b2 = FLT_MAX;                          // best and second-best fp32 distances
  int best = -1;
  for (int j0 = 0; j0 < n; j0 += 4) {
    float4 e[4][LT_EMAX / 128];
    int k[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      k[u] = mi_row[min(j0 + u, n - 1)];
      argmin_load_row(cb + (size_t)k[u] * E, E, lane, e[u]);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (j0 + u < n) {
        float s = 0.f;
#pragma unroll
        for (int q = 0; q < LT_EMAX / 128; ++q) {
          float dd;
          dd = zr[q].x - e[u][q].x; s = fmaf(dd, dd, s);
          dd = zr[q].y - e[u][q].y; s = fmaf(dd, dd, s);
          dd = zr[q].z - e[u][q].z; s = fmaf(dd, dd, s);
          dd = zr[q].w - e[u][q].w; s = fmaf(dd, dd, s);
        }
        s = warp_sum(s);
        if (s < b1 || (s == b1 && k[u] < best)) { b2 = b1; b1 = s; best = k[u]; }
        else if (s < b2) b2 = s;
      }
    }
  }
  // fp32 sums of non-negative terms: relative error <= (2 + 16 + 5) ulp ~ 1.4e-6 each; closer than that -> fp64
  if (!(b1 * (1.f + 4e-6f) < b2)) {
    double bd = 0.0;
    best = -1;
    for (int j = 0; j < n; ++j) {
      const int k = mi_row[j];
      float4 e[LT_EMAX / 128];
      argmin_load_row(cb + (size_t)k * E, E, lane, e);
      double s = 0.0;
#pragma unroll
      for (int q = 0; q < LT_EMAX / 128; ++q) {
        double dd;
        dd = (double)zr[q].x - (double)e[q].x; s += dd * dd;
        dd = (double)zr[q].y - (double)e[q].y; s += dd * dd;
        dd = (double)zr[q].z - (double)e[q].z; s += dd * dd;
        dd = (double)zr[q].w - (double)e[q].w; s += dd * dd;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (best < 0 || s < bd || (s == bd && k < best)) { bd = s; best = k; }
    }
  }
  return best;
}

// per-(token, range, owner) scan results of the split sweep
struct SplitOut {
  int S, per;                  // code ranges, N-tiles per range
  float* win;                  // [T] W of each token
  float* mins;                 // [T][S][2] running minima
  int* cnt;                    // [T][S][2] list lengths (> LT_LIST: overflowed)
  float2* lists;               // [T][S][2][LT_LIST] (d~, code)
};

// ------------------------------------------------------------------------------ the sweep
template <bool SPLIT>
__global__ void __launch_bounds__(LT_THREADS, 1)
l2_argmin_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                    const float* __restrict__ z, const float2* __restrict__ zn2, int T, int E,
                    const float* __restrict__ cb, const float* __restrict__ norm, int K, int64_t* __restrict__ idx,
                    float* __restrict__ quant, int* __restrict__ fb_count, int* __restrict__ fb_list, const SplitOut so) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;                                          // [E/64][128 rows][128 B]: this CTA's 128 tokens
  uint8_t* sB = sA + LT_BM * LT_EMAX * 2;                      // [NST][128 codes][128 B]
  uint8_t* tail = sB + LT_NST * LT_BST;
  float2* lists = reinterpret_cast<float2*>(tail);             // [LT_LIST][2 owners][128 rows] (d~, code)
  float* xmin = reinterpret_cast<float*>(lists + LT_LIST * 2 * LT_BM);   // [2][128] running minima of the two owners
  int* mi = reinterpret_cast<int*>(xmin + 2 * LT_BM);          // [128][LT_TOP] window members
  int* ncand = mi + LT_BM * LT_TOP;                            // [128] members found (zero between tiles)
  int* ovf = ncand + LT_BM;                                    // [128] a list overflowed
  float* xacc = reinterpret_cast<float*>(tail + LT_XCH);       // accumulator exchange
  uint64_t* b_full = reinterpret_cast<uint64_t*>(tail + LT_XCH + LT_XACC);   // [NST]
  uint64_t* b_empty = b_full + LT_NST;                         // [NST]
  uint64_t* a_full = b_empty + LT_NST;                         // [8]
  uint64_t* a_empty = a_full + LT_KBMAX;                       // [8]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int KB = E / LT_BK;                                    // k-blocks
  const int NT = K / LT_BN;                                    // N-tiles
  const int n_t = (T + LT_BM - 1) / LT_BM;                     // 128-token tiles
  // work items: token tiles, or with SPLIT (token tile, code range) pairs, range-minor
  const int n_items = SPLIT ? n_t * so.S : n_t;
  auto item_tile = [&](int wi) { return SPLIT ? wi / so.S : wi; };
  auto item_nt0 = [&](int wi) { return SPLIT ? (wi % so.S) * so.per : 0; };
  auto item_nt1 = [&](int wi) { return SPLIT ? min(NT, (wi % so.S + 1) * so.per) : NT; };

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < LT_NST; ++i) { mbar_init(&b_full[i], 1); mbar_init(&b_empty[i], 8); }
    for (int i = 0; i < LT_KBMAX; ++i) { mbar_init(&a_full[i], 1); mbar_init(&a_empty[i], 8); }
    fence_barrier_init();
  }
  if (threadIdx.x < LT_BM) { ncand[threadIdx.x] = 0; ovf[threadIdx.x] = 0; }
  __syncthreads();

  if (warp == 8) {
    // ---------------------------------------------------------------- codebook producer
    int st = 0;
    uint32_t ph = 0;
    for (int wi = blockIdx.x; wi < n_items; wi += gridDim.x) {
      const int nt1 = item_nt1(wi);
      for (int nt = item_nt0(wi); nt < nt1; ++nt) {
        for (int kb = 0; kb < KB; ++kb) {
          mbar_wait(&b_empty[st], ph ^ 1);
          if (elect_one()) {
            mbar_arrive_expect_tx(&b_full[st], LT_BST);
            tma_load_2d(sB + st * LT_BST, &tmB, &b_full[st], kb * LT_BK, nt * LT_BN);
          }
          __syncwarp();
          if (++st == LT_NST) { st = 0; ph ^= 1; }
        }
      }
    }
  } else if (warp == 9) {
    // ---------------------------------------------------------------- A producer: the bf16 z rows of this CTA's 128 tokens
    int it = 0;
    for (int wi = blockIdx.x; wi < n_items; wi += gridDim.x, ++it) {
      const int t0 = item_tile(wi) * LT_BM;
      for (int kb = 0; kb < KB; ++kb) {
        if (it > 0) mbar_wait(&a_empty[kb], (it - 1) & 1);       // the previous tile's last N-tile has read this k-block
        if (elect_one()) {
          mbar_arrive_expect_tx(&a_full[kb], LT_A_KB_BYTES);
          tma_load_2d(sA + kb * LT_A_KB_BYTES, &tmA, &a_full[kb], kb * LT_BK, t0);       // rows >= T: zero fill
        }
        __syncwarp();
      }
    }
  } else {
    // ---------------------------------------------------------------- 8 worker warps: MMA, scan, merge, exact resolution
    const int w8 = warp;                                       // 0..7
    const int wg = warp >> 2, w = warp & 3;
    const int g = w >> 1;                                      // list owner: which 16 codes of every 32 this thread scans
    const int rl = (w & 1) * 32 + lane;
    const int r = wg * 64 + rl;                                // token row of the tile
    const int bar_id = 2 + wg;                                 // named barrier of this warpgroup's exchange
    float* xw = xacc + wg * 64 * LT_XLD;
    const uint32_t a_rows = smem_u32(sA) + wg * 64 * 128;
    const float emax = sqrtf(__ldg(norm + K)), demax = sqrtf(__ldg(norm + K + 1));
    float2* lst = lists + g * LT_BM + r;
    int st = 0;
    uint32_t ph = 0;
    int it = 0;
    for (int wi = blockIdx.x; wi < n_items; wi += gridDim.x, ++it) {
      const int t0 = item_tile(wi) * LT_BM;
      const int nt0 = item_nt0(wi), nt1 = item_nt1(wi);
      const bool live = t0 + r < T;
      float W;
      {
        const float2 nn = live ? __ldg(zn2 + t0 + r) : make_float2(0.f, 0.f);
        const float zl = sqrtf(nn.x) * 1.0001f, dzl = sqrtf(nn.y) * 1.0001f;
        const float D = 2.f * (dzl * emax + zl * demax) + zl * emax * (1.f / 4096.f) + 1e-30f;
        W = 2.f * D * 1.001f;
      }
      float runmin = live ? FLT_MAX : -FLT_MAX, thr = runmin;  // rows past T never pass the chunk test
      int cnt = 0;
      for (int nt = nt0; nt < nt1; ++nt) {
        float acc[LT_BN / 2];
        int prev = -1;
        for (int kb = 0; kb < KB; ++kb) {
          if (nt == nt0) mbar_wait(&a_full[kb], it & 1);
          mbar_wait(&b_full[st], ph);
          const uint64_t da = wgmma_desc_k_sw128(a_rows + kb * LT_A_KB_BYTES);
          const uint64_t db = wgmma_desc_k_sw128(smem_u32(sB) + st * LT_BST);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < LT_BK / 16; ++k) wgmma_bf16<LT_BN>(acc, da + 2 * k, db + 2 * k, (kb | k) != 0 ? 1u : 0u);
          wgmma_commit();
          wgmma_wait<1>();
          if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&b_empty[prev]); }
          prev = st;
          if (++st == LT_NST) { st = 0; ph ^= 1; }
        }
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) {
          mbar_arrive(&b_empty[prev]);
          if (nt == nt1 - 1)
            for (int kb = 0; kb < KB; ++kb) mbar_arrive(&a_empty[kb]);   // the tile is done with its A k-blocks
        }
        static_for<0, LT_BN / 32>([&](auto rc) {
          constexpr int R = decltype(rc)::value;
          named_bar_sync(bar_id, 128);
          acc_to_smem<32 * R, 32>(acc, xw, LT_XLD, w, lane);
          named_bar_sync(bar_id, 128);
          uint32_t v[LT_SCH];
          const float* src = xw + rl * LT_XLD + g * LT_SCH;
#pragma unroll
          for (int q = 0; q < LT_SCH / 4; ++q) {
            const float4 f = reinterpret_cast<const float4*>(src)[q];
            v[4 * q] = __float_as_uint(f.x); v[4 * q + 1] = __float_as_uint(f.y);
            v[4 * q + 2] = __float_as_uint(f.z); v[4 * q + 3] = __float_as_uint(f.w);
          }
          const int c = nt * LT_BN + 32 * R + g * LT_SCH;
          argmin_scan_chunk(v, norm + c, c, W, smem_u32(lst), runmin, thr, cnt);
        });
      }
      if constexpr (SPLIT) {
        // this range's scan results, merged across ranges by l2_argmin_merge_kernel
        if (live) {
          const int t = t0 + r, s = wi % so.S;
          const size_t o = ((size_t)t * so.S + s) * 2 + g;
          if (s == 0 && g == 0) so.win[t] = W;
          so.mins[o] = runmin;
          so.cnt[o] = cnt;
          for (int j = 0; j < min(cnt, LT_LIST); ++j) so.lists[o * LT_LIST + j] = lst[j * 2 * LT_BM];
        }
        continue;
      }
      // merge: every thread filters its own list against the row's minimum over both owners
      xmin[g * LT_BM + r] = runmin;
      named_bar_sync(1, 256);
      {
        const float win = fminf(xmin[r], xmin[LT_BM + r]) + W;
        if (cnt > LT_LIST) ovf[r] = 1;
        const int nl = min(cnt, LT_LIST);
        for (int j = 0; j < nl; ++j) {
          const float2 e = lst[j * 2 * LT_BM];
          if (e.x <= win) {
            const int pos = atomicAdd(&ncand[r], 1);
            if (pos < LT_TOP) mi[r * LT_TOP + pos] = __float_as_int(e.y);
          }
        }
      }
      named_bar_sync(1, 256);
      // resolution: warp w8 owns rows w8 + 8 i; lane i < 16 looks at row i, windows of one code (the usual case) are done
      // there and then, the others go through the warp-wide exact evaluation one after the other
      {
        const int rr = w8 + 8 * (lane & 15);
        const int t = t0 + rr;
        const bool mine = lane < 16 && t < T;
        int n = 0, best = -1;
        if (mine) {
          n = ncand[rr];
          if (ovf[rr] != 0 || n > LT_TOP || n == 0) n = -1;
          if (n == 1) best = mi[rr * LT_TOP];
          if (n < 0) fb_list[atomicAdd(fb_count, 1)] = t;      // exhaustive kernel
        }
        __syncwarp();
        if (lane < 16) { ncand[rr] = 0; ovf[rr] = 0; }         // only this warp reads these rows: ready for the next tile
        unsigned multi = __ballot_sync(0xffffffffu, mine && n > 1);
        while (multi != 0) {
          const int l = __ffs(multi) - 1;
          multi &= multi - 1;
          const int n_l = __shfl_sync(0xffffffffu, n, l);
          const int rr_l = w8 + 8 * l;
          const int b = argmin_resolve_exact(z, cb, E, t0 + rr_l, n_l, mi + rr_l * LT_TOP, lane);
          if (lane == l) best = b;
        }
        if (mine && n > 0) idx[t] = best;
        if (quant != nullptr) {
          unsigned have = __ballot_sync(0xffffffffu, mine && n > 0);
          while (have != 0) {
            const int l = __ffs(have) - 1;
            have &= have - 1;
            const int b = __shfl_sync(0xffffffffu, best, l);
            const float4* src = reinterpret_cast<const float4*>(cb + (size_t)b * E);
            float4* dst = reinterpret_cast<float4*>(quant + (size_t)(t0 + w8 + 8 * l) * E);
            for (int e = lane; e < (E >> 2); e += 32) dst[e] = __ldg(src + e);
          }
        }
      }
    }
  }

}

// Merge of the split sweep: one warp per token.  Lanes take the (range, owner) lists in turn; entries within W of the
// global minimum are gathered into shared memory in (range, owner, list) order and resolved as in the sweep.
constexpr int LM_WARPS = 8;
__global__ void __launch_bounds__(LM_WARPS * 32)
l2_argmin_merge_kernel(const float* __restrict__ z, int T, int E, const float* __restrict__ cb, const SplitOut so,
                       int64_t* __restrict__ idx, float* __restrict__ quant, int* __restrict__ fb_count,
                       int* __restrict__ fb_list) {
  __shared__ int mi[LM_WARPS][LT_TOP];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t = blockIdx.x * LM_WARPS + warp;
  if (t >= T) return;
  const int nl = 2 * so.S;                                       // lists of this token
  const size_t o0 = (size_t)t * nl;
  float gmin = FLT_MAX;
  bool ovf = false;
  for (int l = lane; l < nl; l += 32) {
    gmin = fminf(gmin, so.mins[o0 + l]);
    ovf |= so.cnt[o0 + l] > LT_LIST;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) gmin = fminf(gmin, __shfl_xor_sync(0xffffffffu, gmin, o));
  ovf = __any_sync(0xffffffffu, ovf);
  const float win = gmin + so.win[t];
  int n = 0;                                                     // window members found so far (warp-uniform)
  for (int l0 = 0; l0 < nl && !ovf; l0 += 32) {
    const int l = l0 + lane;
    const int c = l < nl ? so.cnt[o0 + l] : 0;
    for (int j = 0; j < LT_LIST; ++j) {
      bool in = false;
      int code = 0;
      if (j < c) {
        const float2 e = so.lists[(o0 + l) * LT_LIST + j];
        in = e.x <= win;
        code = __float_as_int(e.y);
      }
      const unsigned m = __ballot_sync(0xffffffffu, in);
      const int pos = n + __popc(m & ((1u << lane) - 1u));
      if (in && pos < LT_TOP) mi[warp][pos] = code;
      n += __popc(m);
    }
  }
  __syncwarp();
  int best;
  if (ovf || n > LT_TOP || n == 0) {
    if (lane == 0) fb_list[atomicAdd(fb_count, 1)] = t;         // exhaustive kernel
    return;
  }
  best = n == 1 ? mi[warp][0] : argmin_resolve_exact(z, cb, E, t, n, mi[warp], lane);
  if (lane == 0) idx[t] = best;
  if (quant != nullptr) {
    const float4* src = reinterpret_cast<const float4*>(cb + (size_t)best * E);
    float4* dst = reinterpret_cast<float4*>(quant + (size_t)t * E);
    for (int e = lane; e < (E >> 2); e += 32) dst[e] = __ldg(src + e);
  }
}

int l2_argmin_list_launch(const float* z, int T, int E, const float* codebook, int K, int64_t* idx, float* quant,
                          const int* list, const int* count, int grid, cudaStream_t st);      // codebook.cu

}  // namespace pgt

using namespace pgt;

extern "C" int pgt_codebook_pack(const float* codebook, int K, int E, void* cb_bf16, float* cb_norm, void* stream) {
  PGT_CHECK_ARG(codebook && cb_bf16 && cb_norm && K > 0 && E > 0);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  PGT_CUDA_OK(cudaMemsetAsync(cb_norm + K, 0, 2 * sizeof(float), st));
  codebook_pack_kernel<<<ceil_div(K, 8), 256, 0, st>>>(codebook, K, E, reinterpret_cast<__nv_bfloat16*>(cb_bf16), cb_norm);
  PGT_LAUNCH_OK();
  return PGT_OK;
}

// workspace layout (int32 units): [fb_count, pad x3][fb_list: T][zn2: T float2][zb: T x LT_EMAX bf16], every section
// 16-byte aligned
static inline int64_t ws_align4(int64_t v) { return (v + 3) & ~int64_t(3); }
static inline int64_t ws_off_list(int T) { (void)T; return 4; }
static inline int64_t ws_off_zn2(int T) { return ws_align4(ws_off_list(T) + T); }
static inline int64_t ws_off_zb(int T) { return ws_align4(ws_off_zn2(T) + (int64_t)T * 2); }

extern "C" int64_t pgt_l2_argmin_ws_ints(int T) {
  return ws_off_zb(T) + (int64_t)T * (LT_EMAX / 2);
}

extern "C" int pgt_l2_argmin_tc(const float* z, int T, int E, const float* codebook, const void* cb_bf16,
                                const float* cb_norm, int K, int64_t* idx, float* quant, int32_t* workspace,
                                void* stream) {
  PGT_CHECK_ARG(z && codebook && cb_bf16 && cb_norm && idx && workspace && T > 0);
  if (K % LT_BN != 0 || E % LT_BK != 0 || E > LT_EMAX || E % 128 != 0) return PGT_ERR_UNSUPPORTED;
  PGT_CHECK_ARG((reinterpret_cast<uintptr_t>(z) & 15) == 0 && (reinterpret_cast<uintptr_t>(codebook) & 15) == 0 &&
                (reinterpret_cast<uintptr_t>(cb_bf16) & 15) == 0 && (reinterpret_cast<uintptr_t>(workspace) & 15) == 0 &&
                (quant == nullptr || (reinterpret_cast<uintptr_t>(quant) & 15) == 0));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int* fb_count = workspace;
  int* fb_list = workspace + ws_off_list(T);
  float2* zn2 = reinterpret_cast<float2*>(workspace + ws_off_zn2(T));
  __nv_bfloat16* zb = reinterpret_cast<__nv_bfloat16*>(workspace + ws_off_zb(T));
  CUtensorMap tmA, tmB;
  int rc = tmap_rows_bf16(&tmA, zb, E, T, E, LT_BM);
  if (rc == PGT_OK) rc = tmap_rows_bf16(&tmB, cb_bf16, E, K, E, LT_BN);
  if (rc != PGT_OK) return rc;
  static PerDeviceOnce once;
  PGT_CUDA_OK(once.run([] { return cudaFuncSetAttribute(l2_argmin_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, LT_SMEM); }));
  PGT_CUDA_OK(cudaMemsetAsync(workspace, 0, sizeof(int32_t), st));
  const int n_t = ceil_div(T, LT_BM);
  const int grid = n_t < num_sms() ? n_t : num_sms();
  {
    ProfScope ps(PGT_PROF_ARGMIN, 2.0 * T * (double)K * E, st, "l2_argmin_tc");
    // pack grid: warps take 4 rows per step; pick the CTA count in [SMs, 2 SMs] that leaves the smallest ragged last step
    int pack_ctas = num_sms() * 2;
    {
      const long long items = ceil_div(T, 4);
      long long best_waste = -1;
      for (int c = num_sms() * 2; c >= num_sms(); --c) {
        const long long w = (long long)c * 8;
        const long long waste = ((items + w - 1) / w) * w - items;
        if (best_waste < 0 || waste < best_waste) { best_waste = waste; pack_ctas = c; }
      }
    }
    z_pack_kernel<<<pack_ctas, 256, 0, st>>>(z, T, E, zb, zn2);
    l2_argmin_tc_kernel<false><<<grid, LT_THREADS, LT_SMEM, st>>>(tmA, tmB, z, zn2, T, E, codebook, cb_norm, K, idx, quant,
                                                                  fb_count, fb_list, SplitOut{});
    PGT_LAUNCH_OK();
  }
  // tokens whose certificate window did not fit the shortlist (degenerate codebooks): exhaustive exact kernel
  return l2_argmin_list_launch(z, T, E, codebook, K, idx, quant, fb_list, fb_count, num_sms(), st);
}

// ------------------------------------------------------------------------------ codebook split (small T)
// workspace (int32 units): the unsplit layout, then [win: T][mins: T x 2S][cnt: T x 2S][lists: T x 2S x LT_LIST float2]
static inline int64_t ws_off_split(int T) { return ws_align4(pgt_l2_argmin_ws_ints(T)); }

static inline int split_ranges(int K, int splits, int* per) {
  const int NT = K / LT_BN;
  const int s = splits < 1 ? 1 : (splits > NT ? NT : splits);
  *per = ceil_div(NT, s);
  return ceil_div(NT, *per);                     // ranges actually used: every one non-empty
}

extern "C" int64_t pgt_l2_argmin_split_ws_ints(int T, int splits) {
  const int64_t L = (int64_t)T * 2 * (splits < 1 ? 1 : splits);
  return ws_off_split(T) + ws_align4(T) + ws_align4(L) + ws_align4(L) + L * LT_LIST * 2;
}

extern "C" int pgt_l2_argmin_tc_split(const float* z, int T, int E, const float* codebook, const void* cb_bf16,
                                      const float* cb_norm, int K, int splits, int64_t* idx, float* quant,
                                      int32_t* workspace, void* stream) {
  PGT_CHECK_ARG(z && codebook && cb_bf16 && cb_norm && idx && workspace && T > 0 && splits >= 1);
  if (K % LT_BN != 0 || E % LT_BK != 0 || E > LT_EMAX || E % 128 != 0) return PGT_ERR_UNSUPPORTED;
  PGT_CHECK_ARG((reinterpret_cast<uintptr_t>(z) & 15) == 0 && (reinterpret_cast<uintptr_t>(codebook) & 15) == 0 &&
                (reinterpret_cast<uintptr_t>(cb_bf16) & 15) == 0 && (reinterpret_cast<uintptr_t>(workspace) & 15) == 0 &&
                (quant == nullptr || (reinterpret_cast<uintptr_t>(quant) & 15) == 0));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int* fb_count = workspace;
  int* fb_list = workspace + ws_off_list(T);
  float2* zn2 = reinterpret_cast<float2*>(workspace + ws_off_zn2(T));
  __nv_bfloat16* zb = reinterpret_cast<__nv_bfloat16*>(workspace + ws_off_zb(T));
  SplitOut so{};
  so.S = split_ranges(K, splits, &so.per);
  // sections sized for `splits` lists per token (>= so.S), so the layout matches pgt_l2_argmin_split_ws_ints
  const int64_t L = (int64_t)T * 2 * splits;
  int32_t* base = workspace + ws_off_split(T);
  so.win = reinterpret_cast<float*>(base);
  so.mins = reinterpret_cast<float*>(base + ws_align4(T));
  so.cnt = base + ws_align4(T) + ws_align4(L);
  so.lists = reinterpret_cast<float2*>(base + ws_align4(T) + 2 * ws_align4(L));
  CUtensorMap tmA, tmB;
  int rc = tmap_rows_bf16(&tmA, zb, E, T, E, LT_BM);
  if (rc == PGT_OK) rc = tmap_rows_bf16(&tmB, cb_bf16, E, K, E, LT_BN);
  if (rc != PGT_OK) return rc;
  static PerDeviceOnce once;
  PGT_CUDA_OK(once.run([] { return cudaFuncSetAttribute(l2_argmin_tc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, LT_SMEM); }));
  PGT_CUDA_OK(cudaMemsetAsync(workspace, 0, sizeof(int32_t), st));
  const int items = ceil_div(T, LT_BM) * so.S;
  const int grid = items < num_sms() ? items : num_sms();
  {
    ProfScope ps(PGT_PROF_ARGMIN, 2.0 * T * (double)K * E, st, "l2_argmin_tc_split");
    z_pack_kernel<<<num_sms() * 2, 256, 0, st>>>(z, T, E, zb, zn2);
    l2_argmin_tc_kernel<true><<<grid, LT_THREADS, LT_SMEM, st>>>(tmA, tmB, z, zn2, T, E, codebook, cb_norm, K, idx, nullptr,
                                                                 fb_count, fb_list, so);
    l2_argmin_merge_kernel<<<ceil_div(T, LM_WARPS), LM_WARPS * 32, 0, st>>>(z, T, E, codebook, so, idx, quant, fb_count,
                                                                            fb_list);
    PGT_LAUNCH_OK();
  }
  return l2_argmin_list_launch(z, T, E, codebook, K, idx, quant, fb_list, fb_count, num_sms(), st);
}
