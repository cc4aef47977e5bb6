// Shifted-window spatio-temporal attention core (WindowAttention3D, modules/rstt_layers.py:195-234, with the roll /
// window_partition / window_reverse / shift mask of VSTSREncoderTransformerBlock :301-329 and EncoderLayer :552-568)
// on TMA + wgmma, sm_90a.
//
// Work unit: a PAIR of 3x4x4 windows (2 x 48 tokens) and one 64-column chunk of the heads (2 heads of d = 32, or one of
// d = 64).  Persistent CTAs, warp-specialised:
//   warp 8     TMA producer.  A window's q / k / v rows of one chunk are ONE 5-D box [64 ch, 4 x, 4 y, 3 frames, clip] of
//              the [T, 3C] qkv matrix (128B swizzle) — the roll by -shift is a coordinate offset, window_partition is the
//              box shape.  Windows in the last window row / column of a shifted block wrap around the frame: they are 2
//              (or 4) half (quarter) boxes, landing one after the other, so their rows sit in a permuted order; attention
//              does not care as long as bias and mask are permuted alike, which the host does once per layer (below).
//              4-deep ring of (k | v | q) chunk tiles.
//   warps 0-3 / 4-7   two warpgroups that alternate chunks.  Per head and window: S = Q K^T as one wgmma 64 x 48 x d
//              (window 0 from tile row 0, window 1 through a view that starts 16 rows before it, so that its 48 rows are
//              rows 16..63 of the MMA), softmax on the register fragments (t = s * scale*log2e + table, exp2, row max and
//              sum across the four lanes of a row), P converted in registers into the A operand of O = P V (wgmma
//              64 x 64 x 16 with A from registers, V read MN-major straight from its TMA tile; for d = 32 the N = 64
//              view spans both heads of the chunk and the other head's half is ignored), then O * (1/sum) -> bf16 -> the
//              token's output row in HBM (window_reverse + roll back are index math).
// Bias / mask table (built at load time by the engine, fp16, already multiplied by log2 e):
//   tab[type][head][j = key/8][row][8]   type 0 interior, 1 x-wrapped (right edge), 2 y-wrapped (bottom edge), 3 corner;
//   entry = relative_position_bias[pi_t(row)][pi_t(key)] + (-100 where the reference's shift mask separates the two
//   tokens), pi_t = the row permutation of the wrapped box order.  Type 0 lives in shared memory, the others in L2.
#include <cuda_fp16.h>

#include "common.cuh"
#include "ptx.cuh"
#include "tmap.cuh"

namespace pgt {

constexpr int WT_N = 48;                          // tokens per window
constexpr int WT_TILE = 2 * WT_N * 128;           // 12 KB: one operand chunk of a window pair (96 rows x 128 B)
constexpr int WT_STAGE = 3 * WT_TILE;             // k | v | q
constexpr int WT_NST = 4;
constexpr int WT_THREADS = 256 + 32;
constexpr int WT_HEADS = 8;
constexpr int WT_TAB_BYTES = WT_HEADS * 6 * WT_N * 16;            // 36 KB: one type of the fp16 table
constexpr int WT_SMEM = 2048 /*pad*/ + WT_NST * WT_STAGE + WT_TAB_BYTES + 512 /*barriers*/ + 1024 /*align*/;

struct WinParams {
  int clips, H, W, C, heads, d, shift;
  int nwx, nwy, n_windows, n_pairs, n_chunks, hpc;   // hpc: heads per 64-column chunk
  int ldo;                                           // output row pitch (elements)
  __nv_bfloat16* out;
  float sl2;                                         // d^-1/2 * log2(e)
  const uint4* tab;                                  // [4][heads][6][48] x 16 B
};

struct WinCoord {
  int clip, x0, y0, xs, ys;        // xs / ys: 1 when the window wraps in x / y
};

__device__ __forceinline__ WinCoord win_coord(const WinParams& p, int w) {
  WinCoord c;
  const int per_clip = p.nwx * p.nwy;
  c.clip = w / per_clip;
  const int r = w - c.clip * per_clip;
  const int wy = r / p.nwx, wx = r - wy * p.nwx;
  c.xs = (p.shift > 0 && wx == p.nwx - 1) ? 1 : 0;
  c.ys = (p.shift > 0 && wy == p.nwy - 1) ? 1 : 0;
  c.x0 = wx * 4 + p.shift;
  c.y0 = wy * 4 + p.shift;
  return c;
}

// Token index (row of the [T, *] matrices) of row `rw` of a window, given its box layout (see the table comment).
__device__ __forceinline__ int win_token(const WinParams& p, const WinCoord& wc, int rw) {
  int f, iy, ix;
  if (!wc.xs && !wc.ys) { f = rw >> 4; iy = (rw >> 2) & 3; ix = rw & 3; }
  else if (wc.xs && !wc.ys) { const int rr = rw % 24; f = rr >> 3; iy = (rr & 7) >> 1; ix = (rr & 1) + 2 * (rw / 24); }
  else if (!wc.xs) { const int rr = rw % 24; f = rr >> 3; iy = ((rr & 7) >> 2) + 2 * (rw / 24); ix = rr & 3; }
  else { const int pp = rw / 12, rr = rw % 12; f = rr >> 2; iy = ((rr & 3) >> 1) + 2 * (pp >> 1); ix = (rr & 1) + 2 * (pp & 1); }
  int y = wc.y0 + iy, x = wc.x0 + ix;                    // rolled coordinates + shift; wrap back into the frame
  if (y >= p.H) y -= p.H;
  if (x >= p.W) x -= p.W;
  return ((wc.clip * 3 + f) * p.H + y) * p.W + x;
}

template <int D>
__global__ void __launch_bounds__(WT_THREADS, 1)
window_attn_tc_kernel(const __grid_constant__ CUtensorMap tmI0, const __grid_constant__ CUtensorMap tmI1,
                      const __grid_constant__ CUtensorMap tmI2, const __grid_constant__ CUtensorMap tmI3,
                      const WinParams p) {
  constexpr int HPC = 64 / D;                                   // heads per 64-column chunk
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* ring = smem + 2048;                                  // [NST][k | v | q] (the window-1 Q view reaches 2 KB back)
  uint8_t* sTab = ring + WT_NST * WT_STAGE;                     // type-0 table
  uint64_t* bars = reinterpret_cast<uint64_t*>(sTab + WT_TAB_BYTES);
  uint64_t* st_full = bars;                                     // [NST]
  uint64_t* st_empty = st_full + WT_NST;                        // [NST] one arrive per warp of the consuming warpgroup

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const CUtensorMap* tmI[4] = {&tmI0, &tmI1, &tmI2, &tmI3};

  if (warp == 8 && lane == 0) {
    for (int i = 0; i < 4; ++i) tma_prefetch_desc(tmI[i]);
    for (int i = 0; i < WT_NST; ++i) { mbar_init(&st_full[i], 1); mbar_init(&st_empty[i], 4); }
    fence_barrier_init();
  }
  // type-0 table -> shared memory (all threads)
  for (int i = threadIdx.x; i < WT_TAB_BYTES / 16; i += WT_THREADS) reinterpret_cast<uint4*>(sTab)[i] = __ldg(p.tab + i);
  __syncthreads();

  const int my_pairs = (p.n_pairs - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;   // pairs blockIdx.x, +gridDim.x, ..
  const int NCH = p.n_chunks;
  const int items = my_pairs * (NCH / 2) * HPC;                 // per warpgroup: (pair, chunk = g mod 2, head in chunk)

  if (warp == 8) {
    // ------------------------------------------------------------------ TMA producer
    int st = 0;
    uint32_t ph = 0;
    for (int i = 0; i < my_pairs; ++i) {
      const int pair = blockIdx.x + i * gridDim.x;
      const int nwin = (2 * pair + 1 < p.n_windows) ? 2 : 1;
      WinCoord wc[2];
      wc[0] = win_coord(p, 2 * pair);
      wc[1] = win_coord(p, nwin == 2 ? 2 * pair + 1 : 2 * pair);
      for (int c = 0; c < NCH; ++c) {
        mbar_wait(&st_empty[st], ph ^ 1);
        if (elect_one()) {
          uint8_t* sK = ring + st * WT_STAGE;
          uint8_t* sV = sK + WT_TILE;
          uint8_t* sQ = sV + WT_TILE;
          mbar_arrive_expect_tx(&st_full[st], nwin * 3 * WT_N * 128);
          for (int wi = 0; wi < nwin; ++wi) {
            const int nx = wc[wi].xs ? 2 : 1, ny = wc[wi].ys ? 2 : 1;
            const CUtensorMap* m = tmI[wc[wi].ys * 2 + wc[wi].xs];
            const int part_bytes = (WT_N / (nx * ny)) * 128;
            int off = wi * WT_N * 128;
            for (int py = 0; py < ny; ++py) {
              const int y = wc[wi].ys ? (py == 0 ? p.H - 2 : 0) : wc[wi].y0;
              for (int px = 0; px < nx; ++px) {
                const int x = wc[wi].xs ? (px == 0 ? p.W - 2 : 0) : wc[wi].x0;
                tma_load_5d(sK + off, m, &st_full[st], p.C + c * 64, x, y, 0, wc[wi].clip);
                tma_load_5d(sQ + off, m, &st_full[st], c * 64, x, y, 0, wc[wi].clip);
                tma_load_5d(sV + off, m, &st_full[st], 2 * p.C + c * 64, x, y, 0, wc[wi].clip);
                off += part_bytes;
              }
            }
          }
        }
        __syncwarp();
        if (++st == WT_NST) { st = 0; ph ^= 1; }
      }
    }
  } else if (warp < 8) {
    // ------------------------------------------------------------------ attention warpgroups
    const int g = warp >> 2;
    const int w = warp & 3;
    const int t4 = lane & 3;
    const int mr = 16 * w + (lane >> 2);                         // MMA rows mr and mr + 8 of this thread (0..63)
    int cur_pair = -1;
    int type[2] = {0, 0};
    __nv_bfloat16* orow[2][2] = {{nullptr, nullptr}, {nullptr, nullptr}};   // [window][row half]
    bool ok[2][2] = {{false, false}, {false, false}};
    int rwin[2][2] = {{0, 0}, {0, 0}};                           // window row of [window][row half] (clamped)

    for (int n = 0; n < items; ++n) {
      const int hh = n % HPC;
      const int cidx = n / HPC;                                  // this warpgroup's chunk counter
      const int pair = blockIdx.x + (cidx / (NCH / 2)) * gridDim.x;
      const int chunk = (cidx % (NCH / 2)) * 2 + g;
      const int head = chunk * HPC + hh;
      const int q = 2 * cidx + g;                                // position of the chunk in the producer's sequence
      const int st = q % WT_NST;
      const uint32_t ph = (q / WT_NST) & 1;
      if (pair != cur_pair) {
        cur_pair = pair;
#pragma unroll
        for (int wi = 0; wi < 2; ++wi) {
          const int wn = 2 * pair + wi;
          const bool win_ok = wn < p.n_windows;
          const WinCoord wc = win_coord(p, win_ok ? wn : 2 * pair);
          type[wi] = wc.ys * 2 + wc.xs;
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int rw = mr + 8 * e - (wi ? 16 : 0);           // window 1 occupies MMA rows 16..63
            ok[wi][e] = win_ok && rw >= 0 && rw < WT_N;
            rwin[wi][e] = rw < 0 ? 0 : (rw >= WT_N ? WT_N - 1 : rw);
            orow[wi][e] = p.out + (size_t)win_token(p, wc, rwin[wi][e]) * p.ldo;
          }
        }
      }
      if (hh == 0) mbar_wait(&st_full[st], ph);
      const uint32_t sK = smem_u32(ring + st * WT_STAGE);
      const uint32_t sV = sK + WT_TILE;
      const uint32_t sQ = sV + WT_TILE;
      const uint32_t koff = hh * D * 2;                          // second head of a d = 32 chunk: +64 B inside the row
#pragma unroll
      for (int wi = 0; wi < 2; ++wi) {
        // ---- S = Q K^T for window wi
        float s[WT_N / 2];
        const uint64_t da = wgmma_desc_k_sw128(sQ + koff + (wi ? (WT_N - 16) * 128 : 0));
        const uint64_t db = wgmma_desc_k_sw128(sK + koff + wi * WT_N * 128);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < D / 16; ++k) wgmma_bf16<WT_N>(s, da + 2 * k, db + 2 * k, k != 0 ? 1u : 0u);
        wgmma_commit();
        // bias / mask of this thread's two rows (type 0 from shared memory, wrapped types from L2) while the MMA runs
        const uint32_t* tb = reinterpret_cast<const uint32_t*>(type[wi] == 0 ? reinterpret_cast<const uint4*>(sTab)
                                                                             : p.tab + (size_t)type[wi] * (WT_TAB_BYTES / 16));
        uint32_t bw[2][6];
#pragma unroll
        for (int e = 0; e < 2; ++e)
#pragma unroll
          for (int j = 0; j < 6; ++j) bw[e][j] = tb[(((size_t)head * 6 + j) * WT_N + rwin[wi][e]) * 4 + t4];
        wgmma_wait<0>();
        // ---- softmax over the 48 keys of each row: 12 per lane, the row's four lanes combine by shuffles
        float mx[2] = {-1e30f, -1e30f};
#pragma unroll
        for (int j = 0; j < 6; ++j) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float2 b2 = __half22float2(*reinterpret_cast<const __half2*>(&bw[e][j]));
            s[4 * j + 2 * e] = fmaf(s[4 * j + 2 * e], p.sl2, b2.x);
            s[4 * j + 2 * e + 1] = fmaf(s[4 * j + 2 * e + 1], p.sl2, b2.y);
            mx[e] = fmaxf(mx[e], fmaxf(s[4 * j + 2 * e], s[4 * j + 2 * e + 1]));
          }
        }
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          mx[e] = fmaxf(mx[e], __shfl_xor_sync(0xffffffffu, mx[e], 1));
          mx[e] = fmaxf(mx[e], __shfl_xor_sync(0xffffffffu, mx[e], 2));
        }
        float sum[2] = {0.f, 0.f};
        uint32_t pa[3][4];                                       // P as the A operand, one k16 step per entry
#pragma unroll
        for (int j = 0; j < 6; ++j) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float e0 = ex2_approx(s[4 * j + 2 * e] - mx[e]), e1 = ex2_approx(s[4 * j + 2 * e + 1] - mx[e]);
            sum[e] += e0 + e1;
            pa[j >> 1][(j & 1) * 2 + e] = pack_bf16x2(e0, e1);
          }
        }
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          sum[e] += __shfl_xor_sync(0xffffffffu, sum[e], 1);
          sum[e] += __shfl_xor_sync(0xffffffffu, sum[e], 2);
        }
        // ---- O = P V (N = 64: the chunk's 64 V columns; d = 32 uses the half of head hh)
        float o[32];
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < WT_N / 16; ++k)
          wgmma_m64n64k16_rs_tb(o, pa[k], wgmma_desc_mn_sw128(sV + (wi * WT_N + k * 16) * 128), k != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
        if (wi == 1 && hh == HPC - 1) {                          // every MMA reading this stage has completed
          __syncwarp();
          if (lane == 0) mbar_arrive(&st_empty[st]);
        }
        // ---- O * (1/sum) -> bf16 -> the token's output row
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          if (!ok[wi][e]) continue;
          const float inv = 1.f / sum[e];
          __nv_bfloat16* dst = orow[wi][e] + chunk * 64 + hh * D + 2 * t4;
#pragma unroll
          for (int j = 0; j < D / 8; ++j) {
            float v0, v1;                                      // columns hh * D + 8 j + 2 t4 (+1)
            if (HPC == 1 || hh == 0) { v0 = o[(j * 4) + 2 * e]; v1 = o[(j * 4) + 2 * e + 1]; }
            else { v0 = o[((D / 8) + j) * 4 + 2 * e]; v1 = o[((D / 8) + j) * 4 + 2 * e + 1]; }
            *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack_bf16x2(v0 * inv, v1 * inv);
          }
        }
      }
    }
  }
}

}  // namespace pgt

using namespace pgt;

// 5-D view [ch, x, y, frame, clip] of a [T, ld] token matrix whose rows are ordered (clip, frame, y, x).
static int win_map(CUtensorMap* map, const void* base, int ld, int cols, int clips, int H, int W, int bx, int by) {
  const uint64_t dims[5] = {(uint64_t)cols, (uint64_t)W, (uint64_t)H, 3, (uint64_t)clips};
  const uint64_t row = (uint64_t)ld * 2;
  const uint64_t strides[4] = {row, row * W, row * W * H, row * W * H * 3};
  const uint32_t box[5] = {64, (uint32_t)bx, (uint32_t)by, 3, 1};
  return tmap_encode(map, base, 5, dims, strides, box);
}

extern "C" int pgt_window_attention_tc(const void* qkv, int ldqkv, int clips, int H, int W, int C, int heads, int shift,
                                       const void* tab, void* out, int ldo, int mode_n64, void* stream) {
  (void)mode_n64;                                           // kept in the ABI: the N = 64 fallback view proved unnecessary
  PGT_CHECK_ARG(qkv && tab && out && clips > 0 && H > 0 && W > 0 && heads > 0);
  PGT_CHECK_ARG(H % 4 == 0 && W % 4 == 0 && C % heads == 0 && ldqkv % 8 == 0 && ldo % 8 == 0 && ldqkv >= 3 * C);
  if (H <= 4 || W <= 4) shift = 0;                         // get_window_size(): no shift when the map is one window
  const int d = C / heads;
  if ((d != 32 && d != 64) || heads != WT_HEADS || C % 128 != 0 || (shift != 0 && shift != 2)) return PGT_ERR_UNSUPPORTED;
  auto al = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  if (!al(qkv) || !al(out) || !al(tab)) return PGT_ERR_UNSUPPORTED;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  CUtensorMap mi[4];
  for (int t = 0; t < 4; ++t) {
    const int bx = (t & 1) ? 2 : 4, by = (t & 2) ? 2 : 4;
    const int rc = win_map(&mi[t], qkv, ldqkv, 3 * C, clips, H, W, bx, by);
    if (rc != PGT_OK) return rc;
  }
  WinParams p{};
  p.clips = clips; p.H = H; p.W = W; p.C = C; p.heads = heads; p.d = d; p.shift = shift;
  p.nwx = W / 4; p.nwy = H / 4;
  p.n_windows = clips * p.nwx * p.nwy;
  p.n_pairs = (p.n_windows + 1) / 2;
  p.n_chunks = C / 64;
  p.hpc = 64 / d;
  p.ldo = ldo;
  p.out = reinterpret_cast<__nv_bfloat16*>(out);
  p.sl2 = (1.0f / sqrtf((float)d)) * 1.4426950408889634f;
  p.tab = reinterpret_cast<const uint4*>(tab);
  const int grid = p.n_pairs < num_sms() ? p.n_pairs : num_sms();
  ProfScope ps(PGT_PROF_WINDOW_ATTN, 4.0 * WT_N * WT_N * C * (double)p.n_windows, st, "window_attn_tc");
  if (d == 32) {
    static PerDeviceOnce once;
    PGT_CUDA_OK(once.run([] { return cudaFuncSetAttribute(window_attn_tc_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, WT_SMEM); }));
    window_attn_tc_kernel<32><<<grid, WT_THREADS, WT_SMEM, st>>>(mi[0], mi[1], mi[2], mi[3], p);
  } else {
    static PerDeviceOnce once;
    PGT_CUDA_OK(once.run([] { return cudaFuncSetAttribute(window_attn_tc_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, WT_SMEM); }));
    window_attn_tc_kernel<64><<<grid, WT_THREADS, WT_SMEM, st>>>(mi[0], mi[1], mi[2], mi[3], p);
  }
  PGT_LAUNCH_OK();
  return PGT_OK;
}
