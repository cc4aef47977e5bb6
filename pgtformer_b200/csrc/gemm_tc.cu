// wgmma GEMM / implicit-GEMM convolution for sm_90a.
//
//   out[rows, N] = epilogue( A[rows, K] * W[N, K]^T )          bf16 operands, fp32 accumulate in registers
//
// Persistent, warp-specialised kernels (384 threads = three warpgroups):
//   warps 0..7  two consumer warpgroups, raised to CONSUMER_REGS registers with setmaxnreg: warpgroup h issues wgmma
//               64 x BN x 16 for rows [64h, 64h + 64) of the 128-row tile over the whole k loop, then runs the epilogue:
//               the accumulators go through a 128 x 64 fp32 shared-memory exchange (one row per thread, 32 columns per
//               chunk) -> +bias -> activation -> +residual / SFT from the staging slot -> optional GroupNorm partial
//               statistics -> bf16/fp32 pack into a 128B-swizzled smem staging panel
//   warps 8..11 warpgroup 2, lowered to PRODUCER_REGS registers:
//     warp 8    TMA producer: A tile (128 rows x 64 K) and W tile (BN rows x 64 K) per k-block, 128B swizzle
//     warp 9    epilogue DMA: TMA-loads the residual (/ SFT scale) panel INTO the staging slot ahead of time and
//               TMA-stores the finished panel, so both are full-line bulk copies and no CTA barrier sits on the path
//     warps 10, 11 idle (setmaxnreg acts on whole warpgroups)
// Pipelines: smem full/empty ring (TMA <-> wgmma) and a staging ring of 4 slots (2 at BN = 256) (epilogue <-> DMA warp);
// the producer runs ahead into the next tile while the consumers finish the epilogue of the current one.
// conv_halo_kernel<BN> runs the consumers PING-PONG instead: each warpgroup owns alternate tiles (all 128 rows)
// and its epilogue (epilogue_tile_wg) runs under the other warpgroup's MMAs.
// Consumer waits do not time out (a reachable trap would hold ptxas to the launch-bound register count); the producer
// and the DMA warp wait with a bound, and the producer ends by waiting until every stage it filled has been released,
// so a transaction that never completes traps the launch instead of hanging it.
//
// Kernels in this file: gemm_tc_kernel<BN> (linear / generic implicit-GEMM conv; BN = 64, 128 or 256),
// conv_halo_kernel<BN> (3x3 and upsample-phase convs with Cout <= 128: one halo slab serves every tap); each also in a
// kVec = false instantiation for bias / output views that are not 16-byte aligned (vector_views).
//
// The A operand is produced by TMA in three addressing modes:
//   LINEAR   2-D map [K, rows]
//   CONV_S1  4-D map [C, W, H, F]; the 128-row tile is a (tn x th x tw) pixel patch and every 3x3 tap is the
//            same box shifted by (dx-1, dy-1); out-of-bounds pixels / channels are zero-filled by TMA, which
//            is exactly the conv zero padding — no im2col buffer, no halo handling in software
//   CONV_S2  5-D map [2C, W/2, 2, H/2, F] (row / column parity split) for stride-2 convs
#include <cudaTypedefs.h>
#include <cstdio>
#include <cstdlib>

#include "common.cuh"
#include "tmap.cuh"
#include "ptx.cuh"
#include "epi_common.cuh"

namespace pgt {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int EPI_WARPS = 8;                     // the two consumer warpgroups (wgmma + epilogue)
constexpr int GEMM_THREADS = EPI_WARPS * 32 + 128;         // consumer warpgroups + the producer / DMA warpgroup
constexpr int PRODUCER_WARP = EPI_WARPS;
constexpr int DMA_WARP = EPI_WARPS + 1;
// setmaxnreg budgets: 2 x 128 x 232 + 128 x 40 = 64512 = 384 x 168, the pool the launch bound gives the CTA
constexpr int CONSUMER_REGS = 232;
constexpr int PRODUCER_REGS = 40;
static_assert(2 * 128 * CONSUMER_REGS + 128 * PRODUCER_REGS <= 65536, "register file");
constexpr int XCH_LD = 68;                       // accumulator exchange: 128 rows x 64 fp32 (+4 pad: conflict-free reads)
constexpr int XCH_BYTES = BM * XCH_LD * 4;
constexpr int XCH_WG_LD = 36;                    // per-warpgroup exchange (ping-pong): 128 rows x 32 fp32 (+4 pad)
constexpr int XCH_WG_BYTES = BM * XCH_WG_LD * 4;
constexpr int EPI_BAR = 1;                       // named barrier of the 256 consumer threads
// ping-pong named barriers, each one per consumer warpgroup h (id + h)
constexpr int PP_XCH_BAR = 2;                    // the warpgroup's 128 threads around its exchange
constexpr int PP_MMA_BAR = 4;                    // "the other warpgroup has issued all MMAs of its tile": h may issue
constexpr int PP_EPI_BAR = 6;                    // "the other warpgroup has finished its epilogue": h may start its own
constexpr int A_STAGE_BYTES = BM * BK * 2;
constexpr int PANEL_BYTES = BM * 128;            // one staging panel: 128 rows x 128 B
// staging slots: 4 (two per epilogue half-group); at BN = 256 a 48 KB stage leaves room for 3 stages and 2 slots
template <int BN>
constexpr int staging_slots() { return BN == 256 ? 2 : 4; }
constexpr int PREFETCH_TILES = 2;                // L2 prefetch distance of the TMA producers, in rounds of gridDim tiles

enum { MODE_LINEAR = 0, MODE_CONV_S1 = 1, MODE_CONV_S2 = 2 };

struct GemmParams {
  int mode;
  int M, N, K;
  int num_kb, m_tiles, n_tiles;
  // conv geometry in OUTPUT space
  int F, H, W;
  int tw, th, tn, tiles_x, tiles_y;
  int cin_blocks, ksize, pad_lo, cin_ld;
  int pad_x, pad_y;            // CONV_S1: zero columns / rows before the first input column / row
  long long o_sx, o_sy, o_sf;  // output element strides of the (x, y, frame) dims (strided placement for up2x)
  // epilogue
  int b_resident;        // halo conv: all 9 weight blocks fit the B ring -> loaded once per CTA, never recycled
  int fast_epi;          // 1: smem-staged TMA-store path, 0: direct per-thread global path
  int has_res_map;       // fast path: residual is TMA-loaded through tmR
  const float* bias;
  int act, epi_mode;
  float* gn_stats;       // optional: per-(tile, group) partial (sum, sumsq) of the OUTPUT for the next GroupNorm(32)
  int gn_cpg;            // channels per group = N / 32
  int ntaps, tap_kw, tap_oy, tap_ox;   // halo conv: 9 taps of a 3x3, or the 4 taps (kw = 2) of an upsample phase at slab offset (oy, ox)
  int gn_tpf;            // > 0: statistics rows are laid out [frame][gn_fstride] (several launches share one buffer)
  int gn_fstride;        //      chunk = (m_blk / gn_tpf) * gn_fstride + (m_blk % gn_tpf) * 4 + quad
  int relu_after_res;    // ResNet BasicBlock: out = relu(conv + shortcut) — ReLU applied after the residual add
  const void* residual;
  int ldr, res_dtype;
  const void* aux;
  int ldaux;
  float sft_w;
  const float* sft_wf;   // conv modes: per-frame fusion weights [F] in place of sft_w (sft_weight), or nullptr
  void* out;
  int ldo, out_dtype, out_layout;
  double flops;      // algorithmic 2*M*N*K with the un-padded K (host-side accounting only)
};

template <int BN>
struct GemmCfg {
  static constexpr int B_STAGE_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  static constexpr int SLOTS = staging_slots<BN>();
  static constexpr int STAGING_BYTES = SLOTS * PANEL_BYTES;
  static constexpr int BUDGET = 232448 - 1024 /*align*/ - STAGING_BYTES - XCH_BYTES - 256 /*barriers*/;
  static constexpr int STAGES = (BUDGET / STAGE_BYTES) > 6 ? 6 : (BUDGET / STAGE_BYTES);
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + STAGING_BYTES + XCH_BYTES + 256 + 1024;
  static_assert(SMEM_BYTES <= 232448, "gemm smem budget");
};

// persistent-loop tile index -> (m block, n block)
__device__ __forceinline__ void tile_mn(const GemmParams& p, int tile, int& m_blk, int& n_blk) {
  n_blk = tile % p.n_tiles;
  m_blk = tile / p.n_tiles;
}


__device__ __forceinline__ void decode_conv_tile(const GemmParams& p, int m_blk, int& n0, int& y0, int& x0) {
  const int tx = m_blk % p.tiles_x;
  const int t2 = m_blk / p.tiles_x;
  const int ty = t2 % p.tiles_y;
  const int tf = t2 / p.tiles_y;
  x0 = tx * p.tw;
  y0 = ty * p.th;
  n0 = tf * p.tn;
}

template <int N>
__device__ __forceinline__ void act_chunk(float (&f)[N], int act) {
  switch (act) {                                  // hoisted: one switch per 32-value chunk
    case PGT_ACT_GELU:
#pragma unroll
      for (int j = 0; j < N; ++j) f[j] = gelu_erf(f[j]);
      break;
    case PGT_ACT_SILU:
#pragma unroll
      for (int j = 0; j < N; ++j) f[j] = apply_act(f[j], PGT_ACT_SILU);
      break;
    case PGT_ACT_LRELU02:
#pragma unroll
      for (int j = 0; j < N; ++j) f[j] = fmaxf(f[j], 0.2f * f[j]);
      break;
    case PGT_ACT_RELU:
#pragma unroll
      for (int j = 0; j < N; ++j) f[j] = fmaxf(f[j], 0.f);
      break;
    case PGT_ACT_SIGMOID:
#pragma unroll
      for (int j = 0; j < N; ++j) f[j] = apply_act(f[j], PGT_ACT_SIGMOID);
      break;
    default: break;
  }
}

// ------------------------------------------------------------------------------------------- epilogue
// Shared by the GEMM/conv kernel and the halo-reuse conv kernel.  Runs on warps 0..7 (256 threads).
struct EpiCtx {
  uint8_t* staging;        // staging_slots<BN>() x PANEL_BYTES, 1024-aligned
  float* xch;              // BM x XCH_LD fp32 accumulator exchange
  uint64_t* res_bar;       // [slots] staging slot prepared (free, residual landed)   DMA warp -> epilogue
  uint64_t* slot_ready;    // [slots] staging slot holds the finished panel           epilogue -> DMA warp
};

// One 32-column chunk of a staging panel, accumulators already in registers (v): +bias -> act -> (+residual | SFT)
// -> packed into the swizzled staging row.  srow is the SHARED-space address of this thread's 128-byte row: explicit
// ld.shared / st.shared (generic LD / ST through the shared window cost several times the latency), and the
// residual vectors are all fetched before the first store so that they overlap instead of serialising behind it.
__device__ __forceinline__ uint4 lds128(uint32_t a) {
  uint4 u;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(u.x), "=r"(u.y), "=r"(u.z), "=r"(u.w) : "r"(a) : "memory");
  return u;
}
__device__ __forceinline__ void sts128(uint32_t a, const uint4& u) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(a), "r"(u.x), "r"(u.y), "r"(u.z), "r"(u.w) : "memory");
}

// SFT fusion weight of the output frame of row r of tile m_blk: sft_wf[frame], or the launch's sft_w.  Rows past the
// last frame (F % tn != 0) are never stored and read the last frame's entry.
__device__ __forceinline__ float sft_weight(const GemmParams& p, int m_blk, int r) {
  if (p.sft_wf == nullptr) return p.sft_w;
  const int f = m_blk / (p.tiles_x * p.tiles_y) * p.tn + r / (p.tw * p.th);
  return __ldg(p.sft_wf + min(f, p.F - 1));
}

template <bool kSft>
__device__ __forceinline__ void epi_finish(const GemmParams& p, const uint32_t (&v)[32], const float* bias32, uint32_t srow,
                                           int r, int sub, int esize, bool has_res, float* gq, int gcol,
                                           const float4 (&pre)[8], bool use_pre, float sw = 0.f) {
  float f[32];
  if (use_pre) {                               // bias chunk already in registers (fetched before the barrier waits)
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      f[4 * q + 0] = __uint_as_float(v[4 * q + 0]) + pre[q].x;
      f[4 * q + 1] = __uint_as_float(v[4 * q + 1]) + pre[q].y;
      f[4 * q + 2] = __uint_as_float(v[4 * q + 2]) + pre[q].z;
      f[4 * q + 3] = __uint_as_float(v[4 * q + 3]) + pre[q].w;
    }
  } else if (bias32 != nullptr) {              // same address in every lane: an L1 broadcast read per float4
    const float4* b4 = reinterpret_cast<const float4*>(bias32);
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const float4 bb = __ldg(b4 + q);
      f[4 * q + 0] = __uint_as_float(v[4 * q + 0]) + bb.x;
      f[4 * q + 1] = __uint_as_float(v[4 * q + 1]) + bb.y;
      f[4 * q + 2] = __uint_as_float(v[4 * q + 2]) + bb.z;
      f[4 * q + 3] = __uint_as_float(v[4 * q + 3]) + bb.w;
    }
  } else {
#pragma unroll
    for (int i = 0; i < 32; ++i) f[i] = __uint_as_float(v[i]);
    if (p.bias != nullptr) {                   // ragged N: guarded scalar reads
#pragma unroll
      for (int i = 0; i < 32; ++i)
        if (gcol + i < p.N) f[i] += __ldg(p.bias + gcol + i);
    }
  }
  if (p.act != PGT_ACT_NONE && !p.relu_after_res) act_chunk(f, p.act);
  if (esize == 2) {
    // 32 bf16 = 64 B = chunks (sub*4 .. sub*4+3) of the 128 B swizzled row
    uint32_t off[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) off[q] = srow + ((((sub << 2) + q) ^ (r & 7)) << 4);
    if (has_res) {
      uint4 ur[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) ur[q] = lds128(off[q]);
      if (kSft) {
        uint4 ux[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) ux[q] = lds128(off[q] + PANEL_BYTES);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float2 a = unpack_bf16x2(ur[q].x), b = unpack_bf16x2(ur[q].y), c = unpack_bf16x2(ur[q].z), d = unpack_bf16x2(ur[q].w);
          const float rr[8] = {a.x, a.y, b.x, b.y, c.x, c.y, d.x, d.y};
          const float2 sa = unpack_bf16x2(ux[q].x), sb = unpack_bf16x2(ux[q].y), sc = unpack_bf16x2(ux[q].z), sd = unpack_bf16x2(ux[q].w);
          const float ss[8] = {sa.x, sa.y, sb.x, sb.y, sc.x, sc.y, sd.x, sd.y};
#pragma unroll
          for (int e = 0; e < 8; ++e) f[8 * q + e] = rr[e] + sw * (rr[e] * ss[e] + f[8 * q + e]);
        }
      } else {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float2 a = unpack_bf16x2(ur[q].x), b = unpack_bf16x2(ur[q].y), c = unpack_bf16x2(ur[q].z), d = unpack_bf16x2(ur[q].w);
          f[8 * q + 0] += a.x; f[8 * q + 1] += a.y; f[8 * q + 2] += b.x; f[8 * q + 3] += b.y;
          f[8 * q + 4] += c.x; f[8 * q + 5] += c.y; f[8 * q + 6] += d.x; f[8 * q + 7] += d.y;
        }
      }
    }
    if (p.relu_after_res) {
#pragma unroll
      for (int e = 0; e < 32; ++e) f[e] = fmaxf(f[e], 0.f);
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      uint4 o;
      o.x = pack_bf16x2(f[8 * q + 0], f[8 * q + 1]);
      o.y = pack_bf16x2(f[8 * q + 2], f[8 * q + 3]);
      o.z = pack_bf16x2(f[8 * q + 4], f[8 * q + 5]);
      o.w = pack_bf16x2(f[8 * q + 6], f[8 * q + 7]);
      sts128(off[q], o);
    }
    if (gq != nullptr) {                       // fused GroupNorm statistics of the (pre-rounding) output values
      const int lane = lane_id();              // re-read, not kept live across the k loop (BN = 256 has no spare registers)
      switch (p.gn_cpg) {
        case 2: gn_chunk_stats<2>(f, gq, 0, lane); break;
        case 4: gn_chunk_stats<4>(f, gq, 0, lane); break;
        case 8: gn_chunk_stats<8>(f, gq, 0, lane); break;
        case 16: gn_chunk_stats<16>(f, gq, 0, lane); break;
        default: gn_chunk_stats<32>(f, gq, 0, lane); break;
      }
    }
  } else {
    // 32 fp32 = 128 B = the whole swizzled row
    if (has_res) {
      uint4 ur[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) ur[q] = lds128(srow + ((q ^ (r & 7)) << 4));
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        f[4 * q + 0] += __uint_as_float(ur[q].x); f[4 * q + 1] += __uint_as_float(ur[q].y);
        f[4 * q + 2] += __uint_as_float(ur[q].z); f[4 * q + 3] += __uint_as_float(ur[q].w);
      }
    }
    if (p.relu_after_res) {
#pragma unroll
      for (int e = 0; e < 32; ++e) f[e] = fmaxf(f[e], 0.f);
    }
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      uint4 o;
      o.x = __float_as_uint(f[4 * q]); o.y = __float_as_uint(f[4 * q + 1]);
      o.z = __float_as_uint(f[4 * q + 2]); o.w = __float_as_uint(f[4 * q + 3]);
      sts128(srow + ((q ^ (r & 7)) << 4), o);
    }
  }
}

// Epilogue work is a stream of ITEMS = (tile, 128-byte-wide column panel) flowing through a ring of staging slots.
// Two roles:
//   * 8 epilogue warps (two per 32-row quadrant, splitting a panel's 32-column chunks; in the ping-pong halo kernel
//     the 4 warps of the tile's warpgroup, one per quadrant, taking both chunks): wait until the slot is
//     prepared, accumulators -> bias / activation / residual / SFT -> swizzled smem, signal `slot_ready`.  No CTA-level
//     barrier and no serial bookkeeping sits on this path.
//   * one DMA warp (epilogue_dma_loop): prepares slots ahead of time (waits for the previous TMA store out of the
//     slot to drain, TMA-loads the residual / SFT-scale panel into it) and TMA-stores finished panels.
struct ItemCursor {
  int tile, pnl;
};

template <int BN>
struct ItemStream {
  const GemmParams& p;
  int num_tiles, PW, panels_total;
  __device__ ItemStream(const GemmParams& pp, int nt) : p(pp), num_tiles(nt) {
    PW = 128 / (pp.out_dtype == PGT_BF16 ? 2 : 4);
    panels_total = BN / PW;
  }
  __device__ int panels_in_tile(int t) const {       // panels whose first column is inside N
    int mb, nb;
    tile_mn(p, t, mb, nb);
    const int cb = nb * BN;
    const int n = (p.N - cb + PW - 1) / PW;
    return n > panels_total ? panels_total : n;
  }
  __device__ bool valid(const ItemCursor& c) const { return c.tile < num_tiles; }
  __device__ void next(ItemCursor& c) const {
    if (++c.pnl >= panels_in_tile(c.tile)) { c.tile += gridDim.x; c.pnl = 0; }
  }
};

template <int BN>
__device__ __forceinline__ void epilogue_dma_loop(const GemmParams& p, const EpiCtx& ctx, const CUtensorMap& tmO,
                                                  const CUtensorMap& tmR, const CUtensorMap& tmX, int lane, int num_tiles) {
  if (!p.fast_epi) return;
  const ItemStream<BN> is(p, num_tiles);
  constexpr int SLOTS = staging_slots<BN>();
  static_assert(SLOTS == 4 || SLOTS == 2, "ring positions are computed with shifts");
  const bool sft = SLOTS == 4 && p.epi_mode == PGT_EPI_SFT;   // dispatch_gemm keeps SFT off the 2-slot ring
  const int S = sft ? 2 : 1;                 // staging slots per item (SFT: residual/out + scale)
  const int R = SLOTS / S;                   // ring length in items: 4, or 2 (SFT, or BN = 256)
  auto coords = [&](const ItemCursor& c, int& col, int& m_blk, int& n0, int& y0, int& x0) {
    int nb;
    tile_mn(p, c.tile, m_blk, nb);
    col = nb * BN + c.pnl * is.PW;
    n0 = y0 = x0 = 0;
    if (p.mode != MODE_LINEAR) decode_conv_tile(p, m_blk, n0, y0, x0);
  };
  // make ring position `pos` ready for item c: its residual (+scale) panel lands there, or it is simply declared free
  auto prepare = [&](const ItemCursor& c, int pos) {
    uint64_t* bar = &ctx.res_bar[pos];
    if (!p.has_res_map) { mbar_arrive(bar); return; }
    int col, m_blk, n0, y0, x0;
    coords(c, col, m_blk, n0, y0, x0);
    uint8_t* dst = ctx.staging + pos * S * PANEL_BYTES;
    mbar_arrive_expect_tx(bar, S * PANEL_BYTES);
    if (p.mode == MODE_LINEAR) {
      tma_load_2d(dst, &tmR, bar, col, m_blk * BM);
      if (sft) tma_load_2d(dst + PANEL_BYTES, &tmX, bar, col, m_blk * BM);
    } else {
      tma_load_4d(dst, &tmR, bar, col, x0, y0, n0);
      if (sft) tma_load_4d(dst + PANEL_BYTES, &tmX, bar, col, x0, y0, n0);
    }
  };
  ItemCursor cp{(int)blockIdx.x, 0}, cs{(int)blockIdx.x, 0};
  if (lane == 0) {
    for (int i = 0; i < R && is.valid(cp); ++i) { prepare(cp, i); is.next(cp); }
  }
  __syncwarp();
  const int rshift = R == 4 ? 2 : 1;                     // no runtime division on this path
  for (int k = 0; is.valid(cs); ++k, is.next(cs)) {
    const int pos = k & (R - 1);
    mbar_wait(&ctx.slot_ready[pos], (k >> rshift) & 1);  // the 8 epilogue warps have written item k
    if (lane == 0) {
      int col, m_blk, n0, y0, x0;
      coords(cs, col, m_blk, n0, y0, x0);
      const uint8_t* src = ctx.staging + pos * S * PANEL_BYTES;
      if (p.mode == MODE_LINEAR) tma_store_2d(&tmO, src, col, m_blk * BM);
      else tma_store_4d(&tmO, src, col, x0, y0, n0);
      bulk_commit();
      // recycle the slot of the PREVIOUS item (for item k-1+R): its store has had a whole item's time to read the panel,
      // so this wait returns at once; waiting for the store just committed (wait_group.read 0) would put a TMA store's
      // issue-to-read latency between consecutive items
      if (k >= 1 && is.valid(cp)) {
        bulk_wait_read<1>();
        prepare(cp, (k - 1) & (R - 1));
        is.next(cp);
      }
    }
    __syncwarp();
  }
  if (lane == 0) bulk_wait0();                           // all output bytes written before the CTA retires
}

// Direct path (NCHW fp32 output, unaligned views, mixed residual dtype): output row of tile row r.
struct DirectRow {
  bool valid;
  long long orow;
  int pn, py, px;
};

__device__ __forceinline__ DirectRow direct_row(const GemmParams& p, int m_blk, int r) {
  DirectRow d{false, 0, 0, 0, 0};
  if (p.mode == MODE_LINEAR) {
    d.orow = (long long)m_blk * BM + r;
    d.valid = d.orow < p.M;
  } else {
    int n0, y0, x0;
    decode_conv_tile(p, m_blk, n0, y0, x0);
    const int ix = r % p.tw;
    const int t2 = r / p.tw;
    const int iy = t2 % p.th;
    const int in = t2 / p.th;
    d.pn = n0 + in; d.py = y0 + iy; d.px = x0 + ix;
    d.valid = (d.pn < p.F) && (d.py < p.H) && (d.px < p.W);
    d.orow = ((long long)d.pn * p.H + d.py) * p.W + d.px;
  }
  return d;
}

// Direct path: columns [col0, col0 + 16) of one output row, accumulators at xs (exchange row), guarded loads / stores.
// kVec: see vector_views.
template <bool kVec>
__device__ __forceinline__ void epi_direct16(const GemmParams& p, const DirectRow& d, const float* xs, int col0) {
  const int ncol = min(16, p.N - col0);
  const long long orow = d.orow;
  float f[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) f[j] = xs[j] + ((p.bias != nullptr && j < ncol) ? __ldg(p.bias + col0 + j) : 0.f);
  if (p.act != PGT_ACT_NONE && !p.relu_after_res) act_chunk(f, p.act);
  if (p.residual != nullptr) {
    if (p.res_dtype == PGT_BF16) {
      const __nv_bfloat16* rp = reinterpret_cast<const __nv_bfloat16*>(p.residual) + orow * p.ldr + col0;
      float rr[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) rr[j] = (j < ncol) ? __bfloat162float(rp[j]) : 0.f;
      if (p.epi_mode == PGT_EPI_SFT) {
        const __nv_bfloat16* ap = reinterpret_cast<const __nv_bfloat16*>(p.aux) + orow * p.ldaux + col0;
        const float sw = p.sft_wf != nullptr ? __ldg(p.sft_wf + d.pn) : p.sft_w;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const float sc = (j < ncol) ? __bfloat162float(ap[j]) : 0.f;
          f[j] = rr[j] + sw * (rr[j] * sc + f[j]);
        }
      } else {
#pragma unroll
        for (int j = 0; j < 16; ++j) f[j] += rr[j];
      }
    } else {
      const float* rp = reinterpret_cast<const float*>(p.residual) + orow * p.ldr + col0;
#pragma unroll
      for (int j = 0; j < 16; ++j)
        if (j < ncol) f[j] += __ldg(rp + j);
    }
  }
  if (p.relu_after_res) act_chunk(f, PGT_ACT_RELU);
  if (p.out_layout == PGT_OUT_NCHW) {
    float* op = reinterpret_cast<float*>(p.out);
#pragma unroll
    for (int j = 0; j < 16; ++j)
      if (j < ncol) op[(((long long)d.pn * p.N + (col0 + j)) * p.H + d.py) * p.W + d.px] = f[j];
  } else if (p.out_dtype == PGT_BF16) {
    __nv_bfloat16* op = reinterpret_cast<__nv_bfloat16*>(p.out) + orow * p.ldo + col0;
    if (kVec && ncol == 16 && ((p.ldo & 7) == 0)) {
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        uint4 u;
        u.x = pack_bf16x2(f[q * 8 + 0], f[q * 8 + 1]);
        u.y = pack_bf16x2(f[q * 8 + 2], f[q * 8 + 3]);
        u.z = pack_bf16x2(f[q * 8 + 4], f[q * 8 + 5]);
        u.w = pack_bf16x2(f[q * 8 + 6], f[q * 8 + 7]);
        reinterpret_cast<uint4*>(op)[q] = u;
      }
    } else {
#pragma unroll
      for (int j = 0; j < 16; ++j)
        if (j < ncol) op[j] = __float2bfloat16_rn(f[j]);
    }
  } else {
    float* op = reinterpret_cast<float*>(p.out) + orow * p.ldo + col0;
#pragma unroll
    for (int j = 0; j < 16; ++j)
      if (j < ncol) op[j] = f[j];
  }
}

// Fused GroupNorm statistics row of (tile m_blk, 32-row quadrant quad) for the chunk starting at column col0.
__device__ __forceinline__ float* gn_stats_ptr(const GemmParams& p, int m_blk, int quad, int col0) {
  if (p.gn_stats == nullptr) return nullptr;
  const size_t chunk = p.gn_tpf > 0 ? (size_t)(m_blk / p.gn_tpf) * p.gn_fstride + (m_blk % p.gn_tpf) * 4 + quad
                                    : (size_t)m_blk * 4 + quad;
  return p.gn_stats + (chunk * 32 + col0 / p.gn_cpg) * 2;
}

// The epilogue of one tile, on the two consumer warpgroups right after their k loop.  Per 64-column group: both
// warpgroups write their accumulator rows into the exchange, then thread (quad, half) reads row quad * 32 + lane,
// columns [32 half, 32 half + 32) (bf16 panels: one chunk each) or the whole panel of parity half (fp32 panels).
// `k` counts staging items across tiles.
template <int BN, bool kVec>
__device__ __forceinline__ void epilogue_tile(const GemmParams& p, const EpiCtx& ctx, int warp, int lane, int tile, int& k,
                                              const float (&acc)[BN / 2]) {
  const int quad = warp & 3;                 // rows [32 quad, 32 quad + 32) of the tile
  const int half = warp >> 2;                // which 32-column chunk of a group / parity of an fp32 panel
  const int r = quad * 32 + lane;            // row of the 128-row tile
  const int esize = (p.out_dtype == PGT_BF16) ? 2 : 4;
  const ItemStream<BN> is(p, 0);
  const int PW = is.PW;
  const int nsub = PW / 32;
  constexpr int SLOTS = staging_slots<BN>();
  constexpr int SLOT_SHIFT = SLOTS == 4 ? 2 : 1;
  const bool sft = SLOTS == 4 && p.epi_mode == PGT_EPI_SFT;
  const bool bias_vec = kVec && p.bias != nullptr && (p.N % 32) == 0;   // whole chunks inside N: 128-bit bias reads
  const float* xrow = ctx.xch + r * XCH_LD;

  int n_blk, m_blk;
  tile_mn(p, tile, m_blk, n_blk);
  const int col_base = n_blk * BN;
  const int npan = p.fast_epi ? is.panels_in_tile(tile) : 0;
  const uint32_t stg = smem_u32(ctx.staging) + r * 128;
  auto gn_ptr = [&](int col0) -> float* { return gn_stats_ptr(p, m_blk, quad, col0); };
  // direct path: this thread's output row
  const DirectRow drow = p.fast_epi ? DirectRow{false, 0, 0, 0, 0} : direct_row(p, m_blk, r);

  static_for<0, BN / 64>([&](auto gc) {
    constexpr int g = decltype(gc)::value;
    if (col_base + g * 64 >= p.N) return;    // uniform over the consumer threads
    named_bar_sync(EPI_BAR, EPI_WARPS * 32);  // the previous group's rows have been read
    acc_to_smem<g * 64, 64>(acc, ctx.xch + half * 64 * XCH_LD, XCH_LD, quad, lane);
    named_bar_sync(EPI_BAR, EPI_WARPS * 32);

    if (p.fast_epi) {
      if (sft) {
        // SFT items (bf16, one panel per group) take two slots (residual / out + scale): ring of 2, one item at a time
        const int pnl = g;
        if (pnl < npan) {
          const int pos = k & 1;
          mbar_wait_spin(&ctx.res_bar[pos], (k >> 1) & 1);   // slot free, residual and scale panels landed
          const int col0 = col_base + pnl * PW + half * 32;
          uint32_t v[32];
          smem_row_32(xrow + half * 32, v);
          float4 nb[8];
          epi_finish<true>(p, v, bias_vec ? p.bias + col0 : nullptr, stg + pos * 2 * PANEL_BYTES, r, half, esize, true,
                           gn_ptr(col0), col0, nb, false, sft_weight(p, m_blk, r));
          fence_proxy_async();                 // generic-proxy smem writes -> visible to the TMA engine
          mbar_arrive(&ctx.slot_ready[pos]);
          ++k;
        }
      } else {
        // One item (panel) at a time; bf16 (two 32-column chunks per panel): the two warpgroups' warps of a quadrant
        // take one chunk each, fp32 (one chunk per panel): they take alternate panels.  The bias chunk is fetched
        // BEFORE the slot wait.
        for (int pp = 0; pp < 64 / PW; ++pp) {
          const int pnl = g * (64 / PW) + pp;
          if (pnl >= npan) break;
          const int pos = k & (SLOTS - 1);
          const bool mine = (nsub == 2) || ((pnl & 1) == half);
          const int sb = (nsub == 2) ? half : 0;
          const int col0 = col_base + pnl * PW + sb * 32;
          float4 b[8];
          const bool pre = BN < 256 && bias_vec;         // BN = 256: no registers to spare, read the bias in epi_finish
          if (mine && pre) {
            const float4* gb = reinterpret_cast<const float4*>(p.bias + col0);
#pragma unroll
            for (int q = 0; q < 8; ++q) b[q] = __ldg(gb + q);
          }
          mbar_wait_spin(&ctx.res_bar[pos], (k >> SLOT_SHIFT) & 1);   // slot free (and residual panel landed)
          if (mine) {
            uint32_t v[32];
            smem_row_32(xrow + pnl * PW + sb * 32 - g * 64, v);
            epi_finish<false>(p, v, bias_vec && !pre ? p.bias + col0 : nullptr, stg + pos * PANEL_BYTES, r, sb, esize,
                              p.has_res_map != 0, gn_ptr(col0), col0, b, pre);
          }
          fence_proxy_async();                 // generic-proxy smem writes -> visible to the TMA engine
          mbar_arrive(&ctx.slot_ready[pos]);
          ++k;
        }
      }
    } else {
      // ---------------- direct path: per-thread global I/O of chunk `half` of the group, 16 columns at a time (the
      // accumulators of the later groups are still live: a 32-wide chunk of guarded loads would not fit beside them)
      const int c0 = g * 64 + half * 32;
      if (drow.valid) {
#pragma unroll 1
        for (int sc16 = 0; sc16 < 32; sc16 += 16) {
          const int col0 = col_base + c0 + sc16;
          if (col0 >= p.N) break;
          epi_direct16<kVec>(p, drow, xrow + half * 32 + sc16, col0);
        }
      }
      __syncwarp();
    }
  });
}

// The epilogue of one tile run by ONE consumer warpgroup (ping-pong schedule: the other warpgroup's MMAs run meanwhile).
// The warpgroup holds all 128 rows as two m64 row blocks, acc[0] = rows [0, 64) and acc[1] = rows [64, 128).  Per
// 32-column chunk: both blocks go through the warpgroup's own 128 x 32 fp32 exchange (ctx.xch), then thread
// (wq, lane) reads row r = 32 wq + lane and finishes it with the same epi_finish / gn_chunk_stats arithmetic as
// epilogue_tile, so outputs and statistics are bit-identical to it.  An item (panel) is signalled to the DMA warp
// once all its chunks are written (slot_ready counts the warpgroup's 128 threads).  `k` is the ring index of the
// tile's first item; `bar` is a named barrier of this warpgroup's 128 threads.
template <int BN, bool kVec>
__device__ __forceinline__ void epilogue_tile_wg(const GemmParams& p, const EpiCtx& ctx, int wq, int bar, int tile, int k,
                                                 const float (&acc)[2][BN / 2]) {
  const int lane = lane_id();                // re-read, not kept live across the k loop (BN = 128 has no spare registers)
  const int r = wq * 32 + lane;
  const int esize = (p.out_dtype == PGT_BF16) ? 2 : 4;
  const ItemStream<BN> is(p, 0);
  const int nsub = is.PW / 32;               // 32-column chunks per panel: 2 (bf16) or 1 (fp32)
  constexpr int SLOTS = staging_slots<BN>();
  constexpr int SLOT_SHIFT = SLOTS == 4 ? 2 : 1;
  const bool sft = SLOTS == 4 && p.epi_mode == PGT_EPI_SFT;    // bf16 only: one 64-column item in two slots
  const bool bias_vec = kVec && p.bias != nullptr && (p.N % 32) == 0;
  const float* xrow = ctx.xch + r * XCH_WG_LD;

  int n_blk, m_blk;
  tile_mn(p, tile, m_blk, n_blk);
  const int col_base = n_blk * BN;
  const int npan = p.fast_epi ? is.panels_in_tile(tile) : 0;
  const uint32_t stg = smem_u32(ctx.staging) + r * 128;
  const DirectRow drow = p.fast_epi ? DirectRow{false, 0, 0, 0, 0} : direct_row(p, m_blk, r);

  static_for<0, BN / 32>([&](auto cc) {
    constexpr int c = decltype(cc)::value;
    const int pnl = c / nsub, sub = c - pnl * nsub;
    if (p.fast_epi && pnl >= npan) return;   // uniform over the warpgroup
    const int col0 = col_base + c * 32;
    if (col0 < p.N) {                        // a chunk wholly past N is clipped by the TMA store: skip its arithmetic
      named_bar_sync(bar, 128);              // the previous chunk's rows have been read
      acc_to_smem<c * 32, 32>(acc[0], ctx.xch, XCH_WG_LD, wq, lane);
      acc_to_smem<c * 32, 32>(acc[1], ctx.xch + 64 * XCH_WG_LD, XCH_WG_LD, wq, lane);
      named_bar_sync(bar, 128);
    }
    if (p.fast_epi) {
      const int item = k + pnl;
      const int pos = sft ? (item & 1) : (item & (SLOTS - 1));
      if (sub == 0) mbar_wait_spin(&ctx.res_bar[pos], sft ? ((item >> 1) & 1) : ((item >> SLOT_SHIFT) & 1));
      if (col0 < p.N) {
        uint32_t v[32];
        smem_row_32(xrow, v);
        float4 nb[8];
        if (sft)
          epi_finish<true>(p, v, bias_vec ? p.bias + col0 : nullptr, stg + pos * 2 * PANEL_BYTES, r, sub, esize, true,
                           gn_stats_ptr(p, m_blk, wq, col0), col0, nb, false, sft_weight(p, m_blk, r));
        else
          epi_finish<false>(p, v, bias_vec ? p.bias + col0 : nullptr, stg + pos * PANEL_BYTES, r, sub, esize,
                            p.has_res_map != 0, gn_stats_ptr(p, m_blk, wq, col0), col0, nb, false);
      }
      if (sub == nsub - 1) {
        fence_proxy_async();                 // generic-proxy smem writes -> visible to the TMA engine
        mbar_arrive(&ctx.slot_ready[pos]);
      }
    } else if (col0 < p.N) {
      if (drow.valid) {
#pragma unroll 1
        for (int sc16 = 0; sc16 < 32; sc16 += 16) {
          if (col0 + sc16 >= p.N) break;
          epi_direct16<kVec>(p, drow, xrow + sc16, col0 + sc16);
        }
      }
      __syncwarp();
    }
  });
}

// Consumer side of a stage ring: one arrive per consumer warp once the warpgroup's wgmmas reading the stage retired.
__device__ __forceinline__ void release_stage(uint64_t* bar, int lane) {
  __syncwarp();
  if (lane == 0) mbar_arrive(bar);
}

template <int BN, bool kVec>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const __grid_constant__ CUtensorMap tmO, const __grid_constant__ CUtensorMap tmR,
               const __grid_constant__ CUtensorMap tmX, const GemmParams p) {
  using Cfg = GemmCfg<BN>;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + STAGES * A_STAGE_BYTES;
  uint8_t* staging = smem + STAGES * Cfg::STAGE_BYTES;                 // 1024-aligned (all stage sizes are)
  float* xch = reinterpret_cast<float*>(staging + Cfg::STAGING_BYTES);
  uint64_t* bars = reinterpret_cast<uint64_t*>(staging + Cfg::STAGING_BYTES + XCH_BYTES);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + STAGES;
  uint64_t* res_bar = bars + 2 * STAGES;                               // [Cfg::SLOTS]
  uint64_t* slot_ready = res_bar + Cfg::SLOTS;                         // [Cfg::SLOTS]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_tiles = p.m_tiles * p.n_tiles;

  if (warp == PRODUCER_WARP && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (p.fast_epi) tma_prefetch_desc(&tmO);
    if (p.has_res_map) tma_prefetch_desc(&tmR);
    if (p.fast_epi && p.epi_mode == PGT_EPI_SFT) tma_prefetch_desc(&tmX);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], EPI_WARPS);       // one arrive per consumer warp
    }
    for (int i = 0; i < Cfg::SLOTS; ++i) {
      mbar_init(&res_bar[i], 1);                 // res_bar / slot_ready: one per staging ring position
      mbar_init(&slot_ready[i], EPI_WARPS * 32);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= EPI_WARPS) {
    setmaxnreg_dec<PRODUCER_REGS>();
    if (warp == PRODUCER_WARP) {
      // ---------------------------------------------------------------- TMA producer
      // (whole warp runs the loop and the waits; the copies are issued under elect.sync so that ptxas sees a
      //  single-lane region and emits the uniform-datapath UTMALDG directly)
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int n_blk, m_blk;
        tile_mn(p, tile, m_blk, n_blk);
        int n0 = 0, y0 = 0, x0 = 0;
        if (p.mode != MODE_LINEAR) decode_conv_tile(p, m_blk, n0, y0, x0);
        for (int kb = 0; kb < p.num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          if (elect_one()) {
            void* dst_a = smem_a + stage * A_STAGE_BYTES;
            void* dst_b = smem_b + stage * Cfg::B_STAGE_BYTES;
            int cb = 0, ax = 0, ay = 0, a5 = 0;            // conv: channel coordinate, x, y (, parity) of this k-block's tap
            if (p.mode != MODE_LINEAR) {
              const int tap = kb / p.cin_blocks;
              cb = kb - tap * p.cin_blocks;
              const int dy = tap / p.ksize;
              const int dx = tap - dy * p.ksize;
              if (p.mode == MODE_CONV_S1) {
                ax = x0 + dx - p.pad_x; ay = y0 + dy - p.pad_y;
              } else {
                const int oy = dy - p.pad_lo, ox = dx - p.pad_lo;
                const int qy = (oy < 0) ? -((1 - oy) >> 1) : (oy >> 1);
                const int qx = (ox < 0) ? -((1 - ox) >> 1) : (ox >> 1);
                const int py = oy - 2 * qy, px = ox - 2 * qx;
                cb = px * p.cin_ld + cb * BK;               // parity-split map: channel coordinate carries the x parity
                ax = x0 + qx; ay = y0 + qy; a5 = py;
              }
            }
            mbar_arrive_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
            if (p.mode == MODE_LINEAR) tma_load_2d(dst_a, &tmA, &full_bar[stage], kb * BK, m_blk * BM);
            else if (p.mode == MODE_CONV_S1) tma_load_4d(dst_a, &tmA, &full_bar[stage], cb * BK, ax, ay, n0);
            else tma_load_5d(dst_a, &tmA, &full_bar[stage], cb, ax, a5, ay, n0);
            tma_load_2d(dst_b, &tmB, &full_bar[stage], kb * BK, n_blk * BN);
          }
          __syncwarp();
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
      // drain: bounded waits until the consumers have released every stage filled above
      for (int i = 0; i < STAGES; ++i) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    } else if (warp == DMA_WARP) {
      // ---------------------------------------------------------------- epilogue DMA warp
      const EpiCtx ctx{staging, xch, res_bar, slot_ready};
      epilogue_dma_loop<BN>(p, ctx, tmO, tmR, tmX, lane, num_tiles);
    }
  } else {
    // ------------------------------------------------------------------ consumer warpgroups: wgmma + epilogue
    setmaxnreg_inc<CONSUMER_REGS>();
    const EpiCtx ctx{staging, xch, res_bar, slot_ready};
    const int wg = warp >> 2;
    const uint32_t a_rows = smem_u32(smem_a) + wg * 64 * 128;        // this warpgroup's 64 rows of every A stage
    const uint32_t b_base = smem_u32(smem_b);
    int stage = 0;
    uint32_t phase = 0;
    int k = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      float acc[BN / 2];
      int prev = -1;
      for (int kb = 0; kb < p.num_kb; ++kb) {
        mbar_wait_spin(&full_bar[stage], phase);
        const uint64_t da = wgmma_desc_k_sw128(a_rows + stage * A_STAGE_BYTES);
        const uint64_t db = wgmma_desc_k_sw128(b_base + stage * Cfg::B_STAGE_BYTES);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < BK / 16; ++kk)           // +32 bytes (2 x 16 B units) per K = 16 step inside the 128 B row
          wgmma_bf16<BN>(acc, da + 2 * kk, db + 2 * kk, (kb | kk) != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();                               // the previous k-block's MMAs have retired: free its stage
        if (prev >= 0) release_stage(&empty_bar[prev], lane);
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      release_stage(&empty_bar[prev], lane);
      epilogue_tile<BN, kVec>(p, ctx, warp, lane, tile, k, acc);
    }
  }
}


// ------------------------------------------------------------------------------------------- halo-reuse conv
// 3x3 stride-1 convolution for narrow outputs (Cout <= 128), where the plain implicit GEMM is bound by
// L2 -> SM traffic (every tap re-reads its 128x64 A tile: 9x input traffic).  Here the 128-pixel tile is a
// 16-row x 8-pixel patch and ONE (16+2) x (8+2) halo slab per 64-channel block serves all nine taps: tap (dy,dx)
// is the same slab viewed from row offset dy*10+dx.  The wgmma descriptor takes the SWIZZLE_128B XOR phase from the
// absolute smem address, as TMA does when it writes the slab, so a K-major operand may start at ANY 128-byte row of
// the slab and its 8-row groups may be any constant stride apart (SBO = slab pitch 1280 B, one image row of 10 pixels).
// A traffic drops from 9 to 1.4 tile-loads per channel block; weights stream through their own ring, or stay
// resident for the whole CTA when all nine taps fit (Cin = 64, Cout <= 64).
constexpr int HALO_TW = 8, HALO_TH = 16;
constexpr int HALO_PITCH = (HALO_TW + 2) * 128;                     // bytes between image rows of the slab
constexpr int HALO_A_BYTES = (HALO_TH + 2) * HALO_PITCH;            // 23040
constexpr int HALO_A_STRIDE = ((HALO_A_BYTES + 1023) / 1024) * 1024; // 23552: keep every slab 1024-aligned

// Each consumer warpgroup has its own accumulator exchange (2 x 18 KB, where one shared exchange takes 34 KB).  At
// BN = 128 that costs a weight stage: the ring keeps 4 of 16 KB instead of 5.  A 3x3 tap of BN = 128 is never resident
// (9 > 5) and the 4-tap upsample phases with Cin <= 64 still are; under the earlier schedule with one shared exchange,
// 4 stages timed the same as 5 on every BN = 128 shape of tools/micro_conv.py halo (H100 80GB HBM3, 700 W).  The
// staging ring keeps its 4 slots, because an SFT item takes two of them.
template <int BN>
struct HaloCfg {
  static constexpr int B_BYTES = BN * 128;
  static constexpr int A_STAGES = 2;
  static constexpr int B_STAGES = (BN == 64) ? 9 : 4;
  static constexpr int SLOTS = staging_slots<BN>();
  static constexpr int STAGING_BYTES = SLOTS * PANEL_BYTES;
  static constexpr int XCH = 2 * XCH_WG_BYTES;
  static constexpr int SMEM_BYTES = A_STAGES * HALO_A_STRIDE + B_STAGES * B_BYTES + STAGING_BYTES + XCH + 512 + 1024;
  static_assert(SMEM_BYTES <= 232448, "halo conv smem budget");
};

// ring position after n more stages of a ring of S
template <int S>
__device__ __forceinline__ void ring_skip(int& s, uint32_t& ph, int n) {
  const int t = s + n;
  ph ^= (uint32_t)(t / S) & 1u;
  s = t % S;
}

template <int BN, bool kVec>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
conv_halo_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const __grid_constant__ CUtensorMap tmO, const __grid_constant__ CUtensorMap tmR,
                 const __grid_constant__ CUtensorMap tmX, const GemmParams p) {
  using Cfg = HaloCfg<BN>;
  constexpr int AS = Cfg::A_STAGES, BS = Cfg::B_STAGES;
  constexpr int RELEASERS = 4;                    // warps releasing a ring stage: the four of the tile's warpgroup
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + AS * HALO_A_STRIDE;
  uint8_t* staging = smem_b + BS * Cfg::B_BYTES;
  float* xch = reinterpret_cast<float*>(staging + Cfg::STAGING_BYTES);
  uint64_t* bars = reinterpret_cast<uint64_t*>(staging + Cfg::STAGING_BYTES + Cfg::XCH);
  uint64_t* a_full = bars;
  uint64_t* a_empty = bars + AS;
  uint64_t* b_full = bars + 2 * AS;
  uint64_t* b_empty = bars + 2 * AS + BS;
  uint64_t* res_bar = bars + 2 * AS + 2 * BS;                          // [Cfg::SLOTS]
  uint64_t* slot_ready = res_bar + Cfg::SLOTS;                         // [Cfg::SLOTS]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_tiles = p.m_tiles * p.n_tiles;
  const int cin_pad = p.cin_blocks * BK;

  if (warp == PRODUCER_WARP && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (p.fast_epi) tma_prefetch_desc(&tmO);
    if (p.has_res_map) tma_prefetch_desc(&tmR);
    if (p.fast_epi && p.epi_mode == PGT_EPI_SFT) tma_prefetch_desc(&tmX);
    for (int i = 0; i < AS; ++i) { mbar_init(&a_full[i], 1); mbar_init(&a_empty[i], RELEASERS); }
    for (int i = 0; i < BS; ++i) { mbar_init(&b_full[i], 1); mbar_init(&b_empty[i], RELEASERS); }
    for (int i = 0; i < Cfg::SLOTS; ++i) {
      mbar_init(&res_bar[i], 1);
      mbar_init(&slot_ready[i], RELEASERS * 32);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= EPI_WARPS) {
    setmaxnreg_dec<PRODUCER_REGS>();
    if (warp == PRODUCER_WARP) {
      // ---------------------------------------------------------------- TMA producer
      int as = 0, bs = 0;
      uint32_t aph = 0, bph = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int n_blk = tile % p.n_tiles;
        const int m_blk = tile / p.n_tiles;
        int n0, y0, x0;
        decode_conv_tile(p, m_blk, n0, y0, x0);
        {
          // pull the slab (and residual panels) of the tile PREFETCH_TILES rounds ahead into L2
          const int pt = tile + PREFETCH_TILES * (int)gridDim.x;
          if (BN == 64 && pt < num_tiles && elect_one()) {
            int pn0, py0, px0;
            decode_conv_tile(p, pt / p.n_tiles, pn0, py0, px0);
            for (int cb = 0; cb < p.cin_blocks; ++cb) tma_prefetch_4d(&tmA, cb * BK, px0 - 1, py0 - 1, pn0);
            if (p.has_res_map) {
              const int c0 = (pt % p.n_tiles) * BN;
              const int rw = p.out_dtype == PGT_BF16 ? 64 : 32;
              for (int c = 0; c < BN && c0 + c < p.N; c += rw) {
                tma_prefetch_4d(&tmR, c0 + c, px0, py0, pn0);
                if (p.epi_mode == PGT_EPI_SFT) tma_prefetch_4d(&tmX, c0 + c, px0, py0, pn0);
              }
            }
          }
          __syncwarp();
        }
        for (int cb = 0; cb < p.cin_blocks; ++cb) {
          mbar_wait(&a_empty[as], aph ^ 1);
          if (elect_one()) {
            mbar_arrive_expect_tx(&a_full[as], HALO_A_BYTES);
            tma_load_4d(smem_a + as * HALO_A_STRIDE, &tmA, &a_full[as], cb * BK, x0 - 1, y0 - 1, n0);
          }
          __syncwarp();
          if (++as == AS) { as = 0; aph ^= 1; }
          if (p.b_resident && tile != (int)blockIdx.x) continue;   // weights already resident in the ring
          for (int t = 0; t < p.ntaps; ++t) {
            mbar_wait(&b_empty[bs], bph ^ 1);
            if (elect_one()) {
              mbar_arrive_expect_tx(&b_full[bs], Cfg::B_BYTES);
              tma_load_2d(smem_b + bs * Cfg::B_BYTES, &tmB, &b_full[bs], t * cin_pad + cb * BK, n_blk * BN);
            }
            __syncwarp();
            if (++bs == BS) { bs = 0; bph ^= 1; }
          }
        }
      }
      // drain: bounded waits until the consumers have released every slab loaded above
      for (int i = 0; i < AS; ++i) {
        mbar_wait(&a_empty[as], aph ^ 1);
        if (++as == AS) { as = 0; aph ^= 1; }
      }
    } else if (warp == DMA_WARP) {
      const EpiCtx ctx{staging, xch, res_bar, slot_ready};
      epilogue_dma_loop<BN>(p, ctx, tmO, tmR, tmX, lane, num_tiles);
    }
  } else {
    // ------------------------------------------------------------------ ping-pong consumer warpgroups
    // The j-th tile of the CTA belongs to warpgroup j & 1, which multiplies all 128 rows (two m64 row blocks on one B
    // descriptor; block 1 = image rows [8, 16) of the patch, 8 slab rows further down) and runs the whole epilogue.
    // Two ordered hand-overs keep the rings and the staging items in tile order:
    //   MMA turn  a warpgroup issues tile j once the other has ISSUED every wgmma of tile j - 1, so the tensor pipe
    //             holds tile j - 1's tail when tile j arrives, and the slab / weight stages are consumed in tile order;
    //   epilogue  it starts the epilogue of tile j once the other has finished that of tile j - 1 (the DMA warp takes
    //             items in order).
    // So one warpgroup's epilogue runs under the other's MMAs.  Each hand-over is a named barrier of 256 threads: the
    // waiting warpgroup syncs, the other arrives, and only when the tile it waits for exists, so none is left pending.
    setmaxnreg_inc<CONSUMER_REGS>();
    const int wg = warp >> 2;
    const EpiCtx ctx{staging, xch + wg * (XCH_WG_BYTES / 4), res_bar, slot_ready};
    const uint32_t a_base = smem_u32(smem_a);
    const uint32_t b_base = smem_u32(smem_b);
    constexpr uint64_t ROW_BLOCK = 8 * HALO_PITCH / 16;   // descriptor units from row block 0 to row block 1
    const ItemStream<BN> is(p, num_tiles);
    const int b_per_tile = p.b_resident ? 0 : p.ntaps * p.cin_blocks;
    int as = 0, bs = 0;
    uint32_t aph = 0, bph = 0;
    int k = 0;
    bool first = true;
    for (int tile = blockIdx.x, j = 0; tile < num_tiles; tile += gridDim.x, ++j) {
      const bool has_next = tile + (int)gridDim.x < num_tiles;
      const int items = p.fast_epi ? is.panels_in_tile(tile) : 0;
      if ((j & 1) != wg) {                             // the other warpgroup's tile: step over its stages and items
        ring_skip<AS>(as, aph, p.cin_blocks);
        ring_skip<BS>(bs, bph, b_per_tile);
        k += items;
        continue;
      }
      if (j > 0) named_bar_sync(PP_MMA_BAR + wg, 256);
      float acc[2][BN / 2];
      for (int cb = 0; cb < p.cin_blocks; ++cb) {
        const bool hand_over = has_next && cb == p.cin_blocks - 1;
        mbar_wait_spin(&a_full[as], aph);
        const uint64_t da0 = wgmma_desc_k_sw128(a_base + as * HALO_A_STRIDE, HALO_PITCH);
        auto tap_desc = [&](int t) -> uint64_t {
          const int dy = t / p.tap_kw, dx = t - dy * p.tap_kw;
          return da0 + (uint64_t)(((dy + p.tap_oy) * (HALO_TW + 2) + dx + p.tap_ox) * 8);
        };
        if (p.b_resident && first) {
          for (int t = 0; t < p.ntaps * p.cin_blocks; ++t) mbar_wait_spin(&b_full[t], 0);
          first = false;
        }
        // One wgmma site for resident and streamed weights: with two, ptxas serialises every wgmma (C7520).
        int prev = -1;
        for (int t = 0; t < p.ntaps; ++t) {
          int bst = cb * p.ntaps + t;                    // resident: the tap's fixed stage
          if (!p.b_resident) {
            mbar_wait_spin(&b_full[bs], bph);
            bst = bs;
          }
          const uint64_t da = tap_desc(t);
          const uint64_t db = wgmma_desc_k_sw128(b_base + bst * Cfg::B_BYTES);
          wgmma_fence();
#pragma unroll
          for (int kk = 0; kk < BK / 16; ++kk) {
            const uint32_t accum = (cb | t | kk) != 0 ? 1u : 0u;
            wgmma_bf16<BN>(acc[0], da + 2 * kk, db + 2 * kk, accum);
            wgmma_bf16<BN>(acc[1], da + ROW_BLOCK + 2 * kk, db + 2 * kk, accum);
          }
          wgmma_commit();
          if (hand_over && t == p.ntaps - 1) named_bar_arrive(PP_MMA_BAR + (wg ^ 1), 256);
          wgmma_wait<1>();                               // the previous tap's weight stage is free
          if (!p.b_resident) {
            if (prev >= 0) release_stage(&b_empty[prev], lane);
            prev = bs;
            if (++bs == BS) { bs = 0; bph ^= 1; }
          }
        }
        wgmma_wait<0>();
        if (!p.b_resident) release_stage(&b_empty[prev], lane);
        release_stage(&a_empty[as], lane);
        if (++as == AS) { as = 0; aph ^= 1; }
      }
      if (j > 0) named_bar_sync(PP_EPI_BAR + wg, 256);
      epilogue_tile_wg<BN, kVec>(p, ctx, warp & 3, PP_XCH_BAR + wg, tile, k, acc);
      if (has_next) named_bar_arrive(PP_EPI_BAR + (wg ^ 1), 256);
      k += items;
    }
  }
}

// ------------------------------------------------------------------------------------------- host side
static int encode_map(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                      const uint32_t* box, int dtype = PGT_BF16) {
  return tmap_encode(map, base, rank, dims, strides_bytes, box, dtype);     // cached (tmap.cuh)
}

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// Output-space tensor map ([N, rows] or [N, W, H, F]) with a 128-byte-wide panel box, for TMA stores of the
// result and TMA loads of the residual.
static int encode_out_map(CUtensorMap* map, const GemmParams& p, const void* base, int ld, int dtype) {
  const int esize = dtype == PGT_BF16 ? 2 : 4;
  const uint32_t pw = 128 / esize;
  if (p.mode == MODE_LINEAR) {
    uint64_t dims[2] = {(uint64_t)p.N, (uint64_t)p.M};
    uint64_t str[1] = {(uint64_t)ld * esize};
    uint32_t box[2] = {pw, BM};
    return encode_map(map, base, 2, dims, str, box, dtype);
  }
  uint64_t dims[4] = {(uint64_t)p.N, (uint64_t)p.W, (uint64_t)p.H, (uint64_t)p.F};
  uint64_t str[3] = {(uint64_t)ld * esize, (uint64_t)p.W * ld * esize, (uint64_t)p.H * p.W * ld * esize};
  if (p.o_sx != 0 && base == p.out) {              // strided placement (only the output map, never the residual)
    str[0] = (uint64_t)p.o_sx * esize; str[1] = (uint64_t)p.o_sy * esize; str[2] = (uint64_t)p.o_sf * esize;
  }
  uint32_t box[4] = {pw, (uint32_t)p.tw, (uint32_t)p.th, (uint32_t)p.tn};
  return encode_map(map, base, 4, dims, str, box, dtype);
}

static int setup_epilogue_maps(GemmParams& p, const CUtensorMap& placeholder, CUtensorMap& tmO, CUtensorMap& tmR,
                               CUtensorMap& tmX) {
  const int esize = p.out_dtype == PGT_BF16 ? 2 : 4;
  p.fast_epi = (p.out_layout == PGT_OUT_NHWC && aligned16(p.out) && ((long long)p.ldo * esize) % 16 == 0) ? 1 : 0;
  if (p.epi_mode == PGT_EPI_SFT &&
      !(p.out_dtype == PGT_BF16 && aligned16(p.aux) && ((long long)p.ldaux * 2) % 16 == 0 && p.o_sx == 0))
    p.fast_epi = 0;
  p.has_res_map = 0;
  if (p.fast_epi && p.residual != nullptr) {
    if (p.res_dtype == p.out_dtype && aligned16(p.residual) && ((long long)p.ldr * esize) % 16 == 0) p.has_res_map = 1;
    else p.fast_epi = 0;
  }
  if (p.gn_stats != nullptr) {
    // fused GroupNorm statistics live on the bf16 TMA-store path; every 128-row tile must sit inside one frame
    const int cpg = p.N / 32;
    const bool ok = p.fast_epi && p.out_dtype == PGT_BF16 && (p.N % 32) == 0 &&
                    (cpg == 2 || cpg == 4 || cpg == 8 || cpg == 16 || cpg == 32) &&
                    (p.mode == MODE_LINEAR || p.tn == 1);
    if (!ok) return PGT_ERR_UNSUPPORTED;
    p.gn_cpg = cpg;
  }
  tmO = placeholder;
  tmR = placeholder;                               // placeholders when unused (never dereferenced)
  tmX = placeholder;
  if (p.fast_epi) {
    int rc = encode_out_map(&tmO, p, p.out, p.ldo, p.out_dtype);
    if (rc != PGT_OK) return rc;
    if (p.has_res_map) {
      rc = encode_out_map(&tmR, p, p.residual, p.ldr, p.res_dtype);
      if (rc != PGT_OK) return rc;
    }
    if (p.epi_mode == PGT_EPI_SFT) {
      if (!p.has_res_map) { p.fast_epi = 0; return p.gn_stats ? PGT_ERR_UNSUPPORTED : PGT_OK; }
      rc = encode_out_map(&tmX, p, p.aux, p.ldaux, PGT_BF16);
      if (rc != PGT_OK) return rc;
    }
  }
  return PGT_OK;
}

// Whether the bias and the output are 16-byte aligned wherever the epilogue accesses them as vectors: the bias of an
// N % 32 == 0 launch (float4 reads) and the bf16 NHWC output of the direct path when ldo % 8 == 0 (uint4 stores).  A view
// starting elsewhere (b + 1, out[:, 1:]) is supported: it runs the kVec = false instantiation of the kernels, whose
// epilogue reads and writes those one element at a time (same values).  Every other call runs kVec = true.
static bool vector_views(const GemmParams& p) {
  if (p.bias != nullptr && (p.N % 32) == 0 && !aligned16(p.bias)) return false;
  if (!p.fast_epi && p.out_layout == PGT_OUT_NHWC && p.out_dtype == PGT_BF16 && (p.ldo % 8) == 0 && !aligned16(p.out))
    return false;
  return true;
}

template <int BN, bool kVec>
static cudaError_t gemm_smem_once() {
  static PerDeviceOnce once;
  return once.run([] {
    return cudaFuncSetAttribute(gemm_tc_kernel<BN, kVec>, cudaFuncAttributeMaxDynamicSharedMemorySize, GemmCfg<BN>::SMEM_BYTES);
  });
}

template <int BN, bool kVec>
static cudaError_t halo_smem_once() {
  static PerDeviceOnce once;
  return once.run([] {
    return cudaFuncSetAttribute(conv_halo_kernel<BN, kVec>, cudaFuncAttributeMaxDynamicSharedMemorySize, HaloCfg<BN>::SMEM_BYTES);
  });
}

static int encode_weight_map(CUtensorMap* tmB, const void* W, int ldw, int K, int N, int BN) {
  // rows beyond N (weight matrices are not padded to BN rows) are zero-filled by TMA
  uint64_t dims[2] = {(uint64_t)K, (uint64_t)N};
  uint64_t str[1] = {(uint64_t)ldw * 2};
  uint32_t box[2] = {BK, (uint32_t)BN};
  return encode_map(tmB, W, 2, dims, str, box);
}

template <int BN>
static int launch_gemm(const CUtensorMap& tmA, const void* W, int ldw, GemmParams& p, cudaStream_t stream) {
  using Cfg = GemmCfg<BN>;
  static_assert(Cfg::STAGES >= 3, "pipeline too shallow");
  CUtensorMap tmB, tmO, tmR, tmX;
  int rc = encode_weight_map(&tmB, W, ldw, p.K, p.N, BN);
  if (rc != PGT_OK) return rc;
  rc = setup_epilogue_maps(p, tmA, tmO, tmR, tmX);
  if (rc != PGT_OK) return rc;
  p.n_tiles = ceil_div(p.N, BN);
  const bool vec = vector_views(p);
  PGT_CUDA_OK((vec ? gemm_smem_once<BN, true>() : gemm_smem_once<BN, false>()));
  const int tiles = p.m_tiles * p.n_tiles;
  const int grid = tiles < num_sms() ? tiles : num_sms();
  {
    char desc[96];
    if (prof_enabled()) {
      if (p.mode == MODE_LINEAR) snprintf(desc, sizeof(desc), "linear M%d N%d K%d BN%d e%d", p.M, p.N, p.K, BN, p.fast_epi);
      else snprintf(desc, sizeof(desc), "conv%d s%d F%d H%d W%d K%d N%d BN%d t%dx%dx%d e%d", p.ksize, p.mode, p.F, p.H, p.W, p.K, p.N, BN, p.tn, p.th, p.tw, p.fast_epi);
    }
    ProfScope ps(PGT_PROF_GEMM, p.flops, stream, desc);
    if (vec) gemm_tc_kernel<BN, true><<<grid, GEMM_THREADS, Cfg::SMEM_BYTES, stream>>>(tmA, tmB, tmO, tmR, tmX, p);
    else gemm_tc_kernel<BN, false><<<grid, GEMM_THREADS, Cfg::SMEM_BYTES, stream>>>(tmA, tmB, tmO, tmR, tmX, p);
  }
  PGT_LAUNCH_OK();
  return PGT_OK;
}

template <int BN>
static int launch_halo(const CUtensorMap& tmA, const void* W, int ldw, GemmParams& p, cudaStream_t stream) {
  using Cfg = HaloCfg<BN>;
  CUtensorMap tmB, tmO, tmR, tmX;
  int rc = encode_weight_map(&tmB, W, ldw, p.K, p.N, BN);
  if (rc != PGT_OK) return rc;
  rc = setup_epilogue_maps(p, tmA, tmO, tmR, tmX);
  if (rc != PGT_OK) return rc;
  p.n_tiles = ceil_div(p.N, BN);
  p.b_resident = (p.ntaps * p.cin_blocks <= Cfg::B_STAGES && p.n_tiles == 1) ? 1 : 0;
  const bool vec = vector_views(p);
  PGT_CUDA_OK((vec ? halo_smem_once<BN, true>() : halo_smem_once<BN, false>()));
  const int tiles = p.m_tiles * p.n_tiles;
  const int grid = tiles < num_sms() ? tiles : num_sms();
  {
    char desc[96];
    if (prof_enabled())
      snprintf(desc, sizeof(desc), "halo3 F%d H%d W%d K%d N%d BN%d e%d r%d", p.F, p.H, p.W, p.K, p.N, BN, p.fast_epi,
               p.b_resident);
    ProfScope ps(PGT_PROF_GEMM, p.flops, stream, desc);
    if (vec) conv_halo_kernel<BN, true><<<grid, GEMM_THREADS, Cfg::SMEM_BYTES, stream>>>(tmA, tmB, tmO, tmR, tmX, p);
    else conv_halo_kernel<BN, false><<<grid, GEMM_THREADS, Cfg::SMEM_BYTES, stream>>>(tmA, tmB, tmO, tmR, tmX, p);
  }
  PGT_LAUNCH_OK();
  return PGT_OK;
}

// Tile width from the shape.  A 128 x 256 tile moves 27 % fewer operand bytes per FLOP than 128 x 128 and reads each
// A tile (every conv tap's) once instead of once per 128 columns; it is used when N > 128 fills whole 256-column tiles
// about as well as 128-column ones, the k loop has at least 8 blocks, and there are enough tiles to occupy every SM.
// Shorter k loops do not amortise the epilogue, which the 2-slot staging ring slows down: on an H100 (400 W) the
// K = 128 / 256 launches of the flagship workload ran 5-12 % slower at BN = 256, every K >= 512 launch 1.0-1.7x faster.
// SFT items take two staging slots and so stay on the 4-slot ring of the 128-wide kernel.
static bool wide_tiles(const GemmParams& p) {
  if (p.N <= 128 || p.num_kb < 8 || p.epi_mode == PGT_EPI_SFT) return false;
  if (ceil_div(p.N, 256) * 256 > ceil_div(p.N, 128) * 128) return false;    // ragged: 256-wide would pad 128 more columns
  return p.m_tiles * ceil_div(p.N, 256) >= num_sms();
}

static int dispatch_gemm(const CUtensorMap& tmA, const void* W, int ldw, GemmParams& p, cudaStream_t stream) {
  if (p.N <= 64) return launch_gemm<64>(tmA, W, ldw, p, stream);
  if (wide_tiles(p)) return launch_gemm<256>(tmA, W, ldw, p, stream);
  return launch_gemm<128>(tmA, W, ldw, p, stream);
}

static int fill_epilogue(GemmParams& p, const pgt_epilogue* ep) {
  if (ep == nullptr || ep->out == nullptr) return PGT_ERR_INVALID;
  p.bias = ep->bias;
  p.act = ep->act;
  p.epi_mode = ep->mode;
  p.residual = ep->residual;
  p.ldr = ep->ldr;
  p.res_dtype = ep->res_dtype;
  p.aux = ep->aux;
  p.ldaux = ep->ldaux;
  p.sft_w = ep->sft_w;
  p.sft_wf = ep->mode == PGT_EPI_SFT ? ep->sft_wf : nullptr;
  p.out = ep->out;
  p.ldo = ep->ldo;
  p.out_dtype = ep->out_dtype;
  p.out_layout = ep->out_layout;
  p.relu_after_res = (ep->flags & PGT_EPI_FLAG_RELU_AFTER_RESIDUAL) ? 1 : 0;
  p.gn_stats = ep->gn_stats;
  p.gn_cpg = 0;
  if (p.relu_after_res && (p.act != PGT_ACT_RELU || p.epi_mode != PGT_EPI_PLAIN)) return PGT_ERR_INVALID;
  if (p.epi_mode == PGT_EPI_SFT && (p.residual == nullptr || p.aux == nullptr || p.res_dtype != PGT_BF16))
    return PGT_ERR_INVALID;
  if (p.sft_wf != nullptr && p.mode == MODE_LINEAR) return PGT_ERR_INVALID;   // a GEMM's rows have no frames
  if (p.out_layout == PGT_OUT_NCHW && (p.out_dtype != PGT_F32 || p.mode == MODE_LINEAR)) return PGT_ERR_INVALID;
  return PGT_OK;
}

}  // namespace pgt

using namespace pgt;

extern "C" int pgt_linear_bf16(const void* A, int lda, const void* W, int ldw, int M, int N, int K,
                               const pgt_epilogue* ep, void* stream) {
  PGT_CHECK_ARG(A && W && M > 0 && N > 0 && K > 0);
  PGT_CHECK_ARG((lda % 8) == 0 && (ldw % 8) == 0 && aligned16(A) && aligned16(W));
  GemmParams p{};
  p.mode = MODE_LINEAR;
  p.M = M; p.N = N; p.K = K;
  p.num_kb = ceil_div(K, BK);
  p.m_tiles = ceil_div(M, BM);
  p.flops = 2.0 * M * (double)N * K;
  int rc = fill_epilogue(p, ep);
  if (rc != PGT_OK) return rc;
  CUtensorMap tmA;
  uint64_t dims[2] = {(uint64_t)K, (uint64_t)M};
  uint64_t str[1] = {(uint64_t)lda * 2};
  uint32_t box[2] = {BK, BM};
  rc = encode_map(&tmA, A, 2, dims, str, box);
  if (rc != PGT_OK) return rc;
  return dispatch_gemm(tmA, W, ldw, p, static_cast<cudaStream_t>(stream));
}

// Tile (tw x th pixels) of a conv of this shape: the 16 x 8 halo tile for the stride-1 3x3 convs (pad 1) and the
// upsample phases (ksize 2, pgt_conv_up2x_bf16) of up to 128 output channels, otherwise the widest power-of-two
// rows of at most 128 pixels.  tw * th < 128 when a 128-row tile spans frames.  Returns whether it is a halo conv.
static bool conv_tile_shape(int Hin, int Win, int Cout, int ksize, int stride, int pad_lo, int& tw, int& th) {
  static const bool no_halo = getenv("PGT_NO_HALO") != nullptr;
  const int H = Hin / stride, W = Win / stride;
  const bool halo = !no_halo && stride == 1 && ((ksize == 3 && pad_lo == 1) || ksize == 2) && Cout <= 128 && Hin >= HALO_TH &&
                    Win >= HALO_TW;
  tw = 1; th = 1;
  if (halo) { tw = HALO_TW; th = HALO_TH; }
  else {
    while (tw * 2 <= W && tw * 2 <= BM) tw *= 2;
    while (th * 2 <= H && tw * th * 2 <= BM) th *= 2;
  }
  return halo;
}

// pad_y/pad_x: zero rows/cols before the input (stride 1); up_phase >= 0: phase (py = up_phase>>1, px = up_phase&1)
// of a nearest-x2-upsample-folded conv — the [F,Hin,Win,Cout] result is scattered to out[F, 2y+py, 2x+px, :].
static int conv_impl(const void* x, int F, int Hin, int Win, int Cin, int ldx, const void* Wp, int ldw, int Cout,
                     int ksize, int stride, int pad_y, int pad_x, int up_phase, const pgt_epilogue* ep, void* stream) {
  const int pad_lo = pad_y;
  PGT_CHECK_ARG(x && Wp && F > 0 && Hin > 0 && Win > 0 && Cin > 0 && Cout > 0);
  PGT_CHECK_ARG((ksize >= 1 && ksize <= 3) && (stride == 1 || stride == 2) && pad_y >= 0 && pad_y <= 1 && pad_x >= 0 && pad_x <= 1);
  PGT_CHECK_ARG(stride == 1 || (ksize != 2 && pad_x == pad_y));
  PGT_CHECK_ARG((ldx % 8) == 0 && (ldw % 8) == 0 && aligned16(x) && aligned16(Wp) && ldx >= Cin);
  const int cin_pad = ceil_div(Cin, BK) * BK;
  PGT_CHECK_ARG(ldw >= ksize * ksize * cin_pad);
  GemmParams p{};
  p.N = Cout;
  p.ksize = ksize;
  p.pad_lo = pad_lo;
  p.pad_x = pad_x; p.pad_y = pad_y;
  p.cin_blocks = cin_pad / BK;
  p.K = ksize * ksize * cin_pad;
  p.num_kb = ksize * ksize * p.cin_blocks;
  p.F = F;
  CUtensorMap tmA;
  int rc;
  if (stride == 1) {
    p.mode = MODE_CONV_S1;
    p.H = Hin; p.W = Win;
  } else {
    if ((Hin & 1) || (Win & 1) || (Cin % BK) != 0 || ldx < Cin) return PGT_ERR_UNSUPPORTED;   // ldx > Cin: channel-slice view of a wider buffer
    p.mode = MODE_CONV_S2;
    p.H = Hin / 2; p.W = Win / 2;
    p.cin_ld = ldx;
  }
  rc = fill_epilogue(p, ep);
  if (rc != PGT_OK) return rc;
  if (up_phase >= 0) {
    if (stride != 1 || p.out_layout != PGT_OUT_NHWC || p.epi_mode != PGT_EPI_PLAIN || p.residual != nullptr)
      return PGT_ERR_UNSUPPORTED;
    const int py = up_phase >> 1, px = up_phase & 1;
    const int esz = p.out_dtype == PGT_BF16 ? 2 : 4;
    const long long Wo = 2LL * Win;
    p.out = static_cast<char*>(p.out) + ((long long)py * Wo + px) * p.ldo * esz;
    p.o_sx = 2LL * p.ldo; p.o_sy = 2LL * Wo * p.ldo; p.o_sf = 4LL * Hin * Win * p.ldo;
  }
  // 128-pixel tile = tn frames x th rows x tw columns (ksize 2 is only ever an upsample phase, and pad_x == pad_y
  // otherwise)
  int tw, th;
  const bool halo = conv_tile_shape(Hin, Win, Cout, ksize, stride, pad_y, tw, th);
  p.ntaps = ksize * ksize; p.tap_kw = ksize;
  p.tap_oy = up_phase >= 0 ? (up_phase >> 1) : 0;          // phase (py, px): tap (dy, dx) reads slab row dy + py, col dx + px
  p.tap_ox = up_phase >= 0 ? (up_phase & 1) : 0;
  const int tn = BM / (tw * th);
  p.tw = tw; p.th = th; p.tn = tn;
  p.tiles_x = ceil_div(p.W, tw);
  p.tiles_y = ceil_div(p.H, th);
  p.m_tiles = p.tiles_x * p.tiles_y * ceil_div(F, tn);
  p.M = F * p.H * p.W;
  p.flops = 2.0 * p.M * (double)Cout * (ksize * ksize * Cin);
  if (up_phase >= 0 && p.gn_stats != nullptr) {
    // the four phase launches share one statistics buffer [frame][phase][tile][quadrant][32][2]
    if (tn != 1) return PGT_ERR_UNSUPPORTED;
    const int tpf = p.tiles_x * p.tiles_y;
    p.gn_tpf = tpf;
    p.gn_fstride = 16 * tpf;
    p.gn_stats += (size_t)up_phase * tpf * 4 * 64;
  }
  if (p.mode == MODE_CONV_S1) {
    uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)Win, (uint64_t)Hin, (uint64_t)F};
    uint64_t str[3] = {(uint64_t)ldx * 2, (uint64_t)Win * ldx * 2, (uint64_t)Hin * Win * ldx * 2};
    uint32_t box[4] = {BK, (uint32_t)(halo ? tw + 2 : tw), (uint32_t)(halo ? th + 2 : th), (uint32_t)tn};
    rc = encode_map(&tmA, x, 4, dims, str, box);
    if (rc == PGT_OK && halo) {
      cudaStream_t st = static_cast<cudaStream_t>(stream);
      return Cout <= 64 ? launch_halo<64>(tmA, Wp, ldw, p, st) : launch_halo<128>(tmA, Wp, ldw, p, st);
    }
  } else {
    uint64_t dims[5] = {(uint64_t)2 * ldx, (uint64_t)Win / 2, 2, (uint64_t)Hin / 2, (uint64_t)F};
    uint64_t str[4] = {(uint64_t)2 * ldx * 2, (uint64_t)Win * ldx * 2, (uint64_t)2 * Win * ldx * 2,
                       (uint64_t)Hin * Win * ldx * 2};
    uint32_t box[5] = {BK, (uint32_t)tw, 1, (uint32_t)th, (uint32_t)tn};
    rc = encode_map(&tmA, x, 5, dims, str, box);
  }
  if (rc != PGT_OK) return rc;
  if (up_phase >= 0) {
    // strided placement exists only on the TMA-store path
    const int esz = p.out_dtype == PGT_BF16 ? 2 : 4;
    if (!aligned16(p.out) || ((long long)p.ldo * esz) % 16 != 0) return PGT_ERR_UNSUPPORTED;
  }
  return dispatch_gemm(tmA, Wp, ldw, p, static_cast<cudaStream_t>(stream));
}

// 128-row tiles per frame of the conv the library would launch for this shape (0: a tile may span frames, so the
// fused GroupNorm statistics are unavailable).
extern "C" int pgt_conv_tiles_per_frame(int Hin, int Win, int Cout, int ksize, int stride, int pad_lo) {
  int tw, th;
  conv_tile_shape(Hin, Win, Cout, ksize, stride, pad_lo, tw, th);
  if (tw * th != BM) return 0;
  return ceil_div(Win / stride, tw) * ceil_div(Hin / stride, th);
}

// The same, and 0 also when the tile grid does not divide the frame: the epilogue sums all 128 rows of a tile into the
// statistics, so a tile that reaches past the frame's right or bottom edge adds rows that are not output pixels.
extern "C" int pgt_conv_tiles_exact(int Hin, int Win, int Cout, int ksize, int stride, int pad_lo) {
  int tw, th;
  conv_tile_shape(Hin, Win, Cout, ksize, stride, pad_lo, tw, th);
  if (tw * th != BM) return 0;
  const int H = Hin / stride, W = Win / stride;
  return (W % tw == 0 && H % th == 0) ? (W / tw) * (H / th) : 0;
}

extern "C" int pgt_conv_bf16(const void* x, int F, int Hin, int Win, int Cin, int ldx, const void* Wp, int ldw,
                             int Cout, int ksize, int stride, int pad_lo, const pgt_epilogue* ep, void* stream) {
  PGT_CHECK_ARG(ksize == 1 || ksize == 3);
  return conv_impl(x, F, Hin, Win, Cin, ldx, Wp, ldw, Cout, ksize, stride, pad_lo, pad_lo, -1, ep, stream);
}

extern "C" int pgt_conv_up2x_bf16(const void* x, int F, int Hin, int Win, int Cin, int ldx, const void* Wp4, int ldw,
                                  int Cout, const pgt_epilogue* ep, void* stream) {
  PGT_CHECK_ARG(Wp4 != nullptr && ldw > 0);
  const int cin_pad = ceil_div(Cin, BK) * BK;
  PGT_CHECK_ARG(ldw >= 4 * cin_pad);
  for (int ph = 0; ph < 4; ++ph) {
    const int py = ph >> 1, px = ph & 1;
    const void* w = static_cast<const char*>(Wp4) + (size_t)ph * Cout * ldw * 2;
    int rc = conv_impl(x, F, Hin, Win, Cin, ldx, w, ldw, Cout, 2, 1, 1 - py, 1 - px, ph, ep, stream);
    if (rc != PGT_OK) return rc;
  }
  return PGT_OK;
}
