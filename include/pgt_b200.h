/* pgt_b200.h — C ABI of libpgt_b200.so: the hand-written sm_90a kernels behind
 * PGTFormer.forward.
 *
 * The reference (kepengxu/PGTFormer) exposes a Python class and no FFI (SURVEY.md 8b); these
 * entry points are what a `torch.ops`/ctypes binding for the hot path would bind.  Each entry
 * cites the reference code it replaces (paths relative to the reference repository).
 *
 * Conventions
 *  - every function returns 0 (PGT_OK) or a negative pgt_status; it never throws, never
 *    synchronises the device and never allocates caller-visible memory;
 *  - all pointers are DEVICE pointers unless stated otherwise; `stream` is a cudaStream_t;
 *  - activations are channels-last: a feature map is [F, H, W, C] (F = clips*3 frames) with an
 *    explicit row stride `ld*` in ELEMENTS (so a kernel can read/write a channel slice of a wider
 *    buffer); token matrices are [T, C] row-major.  bf16 unless a `*_dtype` argument says fp32;
 *  - weights are pre-packed once at load time (pgtformer_b200/engine.py): linear [N, K] bf16 row
 *    major; conv [Cout, taps*CinPad] bf16 with K index = tap*CinPad + c, CinPad = roundup(Cin, 64).
 */
#ifndef PGT_B200_H_
#define PGT_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum pgt_status {
  PGT_OK = 0,
  PGT_ERR_INVALID = -1,      /* bad shape / alignment / null pointer                      */
  PGT_ERR_CUDA = -2,         /* a CUDA runtime call failed (see pgt_last_cuda_error)       */
  PGT_ERR_UNSUPPORTED = -3,  /* valid request the sm_90a kernels do not cover             */
  PGT_ERR_DRIVER = -4        /* cuTensorMapEncodeTiled unavailable / failed               */
} pgt_status;

enum { PGT_BF16 = 0, PGT_F32 = 1 };
enum { PGT_ACT_NONE = 0, PGT_ACT_GELU = 1, PGT_ACT_SILU = 2, PGT_ACT_LRELU02 = 3, PGT_ACT_RELU = 4,
       PGT_ACT_SIGMOID = 5 };
enum { PGT_EPI_PLAIN = 0,    /* y = act(acc + bias) [+ residual]                           */
       PGT_EPI_SFT = 1 };    /* y = r + w * (r * aux + (acc + bias)); r = residual         */
enum { PGT_OUT_NHWC = 0, PGT_OUT_NCHW = 1 };
/* act must be PGT_ACT_RELU: y = relu(acc + bias + residual)  (ResNet BasicBlock, archs/pgtformer_arch.py:56-68) */
enum { PGT_EPI_FLAG_RELU_AFTER_RESIDUAL = 1 };

/* Fused epilogue shared by the tensor-core GEMM / implicit-GEMM conv. */
typedef struct pgt_epilogue {
  const float* bias;     /* [N] fp32 or NULL                                               */
  int32_t act;           /* PGT_ACT_*                                                      */
  int32_t mode;          /* PGT_EPI_*                                                      */
  const void* residual;  /* optional [rows, ldr]                                           */
  int32_t ldr;
  int32_t res_dtype;     /* PGT_BF16 / PGT_F32                                             */
  const void* aux;       /* PGT_EPI_SFT: scale tensor, bf16 [rows, ldaux]                  */
  int32_t ldaux;
  float sft_w;           /* PGT_EPI_SFT: fusion weight w                                   */
  void* out;             /* [rows, ldo] (NHWC) or [F, N, H, W] (NCHW, conv only)           */
  int32_t ldo;
  int32_t out_dtype;     /* PGT_BF16 / PGT_F32                                             */
  int32_t out_layout;    /* PGT_OUT_NHWC / PGT_OUT_NCHW                                    */
  int32_t flags;         /* PGT_EPI_FLAG_*                                                  */
  float* gn_stats;       /* optional fp32 [rows/128, 4, 32, 2]: per-(tile, 32-row quadrant) (sum, sumsq) of the output per GroupNorm(32)
                          * group, produced by the epilogue for the NEXT Normalize() (bf16 NHWC output, N % 32 == 0,
                          * every 128-row tile inside one frame: pgt_conv_tiles_per_frame() > 0 (exact statistics:
                          * pgt_conv_tiles_exact() > 0), or HW % 128 == 0 for
                          * pgt_linear_bf16); consumed by pgt_groupnorm_apply_stats                         */
} pgt_epilogue;

const char* pgt_strerror(int status);
const char* pgt_last_cuda_error(void);
int pgt_version(void);
/* Number of kernel launches issued through this library since the last reset (bench.py's
 * `gpu_launches` claim). */
int64_t pgt_launch_count(void);
void pgt_reset_launch_count(void);
/* CUtensorMap cache (one encode per distinct (pointer, shape, box) for the life of the process): hit / miss counters. */
void pgt_tmap_cache_stats(int64_t* hits, int64_t* misses);

/* Optional per-launch profiler (bench.py's roofline figures): between begin and end every launch of
 * the classes below is bracketed by CUDA events on its own stream; end() synchronises and returns,
 * per class, the summed algorithmic work (FLOPs, or bytes for the HBM-bound classes), the summed
 * device time in ms and the launch count.  Arrays have PGT_PROF_CLASSES entries. */
enum { PGT_PROF_GEMM = 0, PGT_PROF_WINDOW_ATTN = 1, PGT_PROF_MHA = 2, PGT_PROF_ARGMAX = 3, PGT_PROF_ARGMIN = 4,
       PGT_PROF_NORM = 5, PGT_PROF_MOVE = 6, PGT_PROF_LAYERNORM = 7, PGT_PROF_CLASSES = 8 };
int pgt_profile_begin(void);
int pgt_profile_end(double* work, double* ms, int64_t* launches);
/* same, and also writes one CSV row per launch (class, description, work, ms) to `path` (host string). */
int pgt_profile_end_csv(const char* path, double* work, double* ms, int64_t* launches);

/* ---- wgmma GEMM:  out[M,N] = epilogue(A[M,K] * W[N,K]^T)
 * Replaces nn.Linear / 1x1 Conv2d call sites: WindowAttention3D q/kv/proj
 * (modules/rstt_layers.py:210-212,231), Mlp fc1/fc2 (:126-131), nn.MultiheadAttention in/out
 * projections and linear1/linear2 (archs/codeformer_arch.py:105-108,127-136), feat_emb /
 * idx_pred_layer (archs/pgtformer_arch.py:520-533), quant_conv / post_quant_conv
 * (archs/tdcrqvae3_arch.py:754-755), convpos, nin_shortcut, SFT 1x1 mixers
 * (archs/pgtformer_arch.py:454-458).  lda, ldw multiples of 8; A, W 16-byte aligned. */
int pgt_linear_bf16(const void* A, int lda, const void* W, int ldw, int M, int N, int K,
                    const pgt_epilogue* ep, void* stream);

/* ---- wgmma implicit-GEMM convolution on NHWC bf16.
 * ksize in {1,3}; stride in {1,2}; pad_lo = zero rows/cols before the first input row/col
 * (3x3 s1: 1; Downsample pad(0,1,0,1): 0; ResNet 3x3 s2: 1), the far side is zero-filled as
 * needed.  Output is [F, Hout, Wout, Cout], Hout = Hin/stride.
 * Replaces Conv2d 3x3 in TDResnetBlock (modules/rstt_layers.py:875-904), ResBlock / scale / shift
 * (archs/pgtformer_arch.py:421-432,442-450), Upsample.conv / Downsample.conv
 * (archs/tdcrqvae3_arch.py:45-52,67-76), conv_in/conv_out, and the BiSeNet convs. */
int pgt_conv_bf16(const void* x, int F, int Hin, int Win, int Cin, int ldx, const void* Wp, int ldw,
                  int Cout, int ksize, int stride, int pad_lo, const pgt_epilogue* ep, void* stream);

/* ---- decoder tail: GroupNorm(32) -> SiLU -> 3x3 conv to <= 3 channels -> fp32 NCHW, one wgmma kernel (conv_out.cu).
 * x: RAW (pre-norm) bf16 [F, H, W, 64]; gn_ab: fp32 [F][2][64] from pgt_groupnorm_ab; Wp: packed [Cout, 9*64] bf16;
 * out: fp32 [F, Cout, H, W].  Replaces norm_out / nonlinearity / conv_out at the end of the decoder
 * (archs/pgtformer_arch.py:707-710, archs/tdcrqvae3_arch.py:700-706).  PGT_ERR_UNSUPPORTED unless Cin == 64,
 * Cout <= 3, H % 16 == 0, W % 8 == 0. */
int pgt_conv_out_gn(const void* x, int F, int H, int W, int Cin, int ldx, const float* gn_ab, const void* Wp, int ldw,
                    int Cout, const float* bias, float* out, void* stream);
/* The same with the activation chosen: silu = 1 is pgt_conv_out_gn (same kernel, same bits); silu = 0 is
 * GroupNorm -> conv with no SiLU, the end of VQGAN's / CodeFormer's generator (archs/vqgan_arch.py:329-332). */
int pgt_conv_out_gn_act(const void* x, int F, int H, int W, int Cin, int ldx, const float* gn_ab, const void* Wp, int ldw,
                        int Cout, const float* bias, float* out, int silu, void* stream);

/* ---- GroupNorm(32)+SiLU of the INPUT fused into the 3x3 / stride 1 / pad 1 conv: the normalised activation is never
 * written to HBM — the kernel applies y = silu(x * a[f,c] + b[f,c]) to each input slab in shared memory (bit-identical
 * to pgt_groupnorm_silu's apply pass) before the MMAs read it.  gn_ab: fp32 [F][2][Cin] from pgt_groupnorm_ab.
 * Available where the halo-reuse kernel is (pgt_conv_gn_supported: Cout <= 128, Hin >= 16, Win >= 8, Cin % 8 == 0);
 * PGT_ERR_UNSUPPORTED otherwise.  Replaces  Normalize -> swish -> conv  of TDResnetBlock (modules/rstt_layers.py:
 * 875-904), ResBlock (archs/pgtformer_arch.py:421-432) and norm_out -> conv_out (archs/tdcrqvae3_arch.py:569-572). */
int pgt_conv_gn_supported(int Hin, int Win, int Cin, int Cout);
int pgt_conv_gn_bf16(const void* x, int F, int Hin, int Win, int Cin, int ldx, const float* gn_ab, const void* Wp,
                     int ldw, int Cout, const pgt_epilogue* ep, void* stream);

/* ---- nearest-x2 upsample + 3x3 conv as ONE op, without materialising the upsampled tensor: the output
 * pixel (2y+py, 2x+px) only sees a 2x2 neighbourhood of the source, so the op is four 2x2 convolutions
 * (one per output phase) over the SOURCE resolution with tap-summed weights: 4/9 of the FLOPs, 1/4 of the
 * A traffic.  Wp4: bf16 [4 phases][Cout][4*CinPad], phase = py*2+px, K index = (ty*2+tx)*CinPad + c, where
 * taps of phase p are the sums w[Sy(ty), Sx(tx)] with S(0) = {0} / {0,1} and S(1) = {1,2} / {2} for p = 0 / 1
 * (packed by pgtformer_b200/engine.py::_pack_up2x).  ep->out is the [F, 2Hin, 2Win, Cout] result.
 * ep->gn_stats (optional): fp32 [F][4 phases][tiles per phase-frame][4][32][2], i.e. 16 * tiles chunks per frame
 * with tiles = pgt_conv_tiles_per_frame(Hin, Win, Cout, 2, 1, 1).
 * Replaces Upsample.forward (archs/tdcrqvae3_arch.py:45-52). */
int pgt_conv_up2x_bf16(const void* x, int F, int Hin, int Win, int Cin, int ldx, const void* Wp4, int ldw,
                       int Cout, const pgt_epilogue* ep, void* stream);

/* ---- the two Cin = 3 convolutions on the tensor cores, reading the fp32 NCHW image directly (im2col inside the
 * kernel): ksize/stride/pad = 3/1/1 (Encoder.conv_in, archs/tdcrqvae3_arch.py:500-504) or 7/2/3 (Resnet18.conv1 +
 * folded bn1 + relu, archs/pgtformer_arch.py:95-99,110-112); Cout = 64.
 *   Wp: bf16 [Cout, ldw], K index (ky*ksize + kx)*3 + c, ldw % 8 == 0;  mean3 / std3: HOST pointers to 3 floats or
 *   NULL: the input is (x - mean) / std with zero padding applied after the normalisation, as in the reference;
 *   act: PGT_ACT_NONE or PGT_ACT_RELU;  out: bf16 [F*Ho*Wo, ldo];  gn_stats: optional GroupNorm partials of the
 *   output, fp32 [ceil(F*Ho*Wo/128)][4][32][2] (requires Ho*Wo % 128 == 0).
 * PGT_ERR_UNSUPPORTED for any other geometry. */
int pgt_conv_rgb_bf16(const float* x_nchw, int F, int H, int W, int ksize, int stride, int pad, const float* mean3,
                      const float* std3, const void* Wp, int ldw, int Cout, const float* bias, int act, void* out,
                      int ldo, float* gn_stats, void* stream);

/* ---- GroupNorm(32, eps) [+ SiLU] on NHWC bf16: y = act((x-mean)*rstd*gamma+beta).
 * `ws` is a caller-provided fp32 workspace of at least pgt_groupnorm_ws_floats(F, HW, C) floats.
 * Replaces Normalize()+nonlinearity (modules/rstt_layers.py:754-758,880-881,889-890) and
 * normalize()+swish (archs/pgtformer_arch.py:406-407,423-428). */
int64_t pgt_groupnorm_ws_floats(int F, int HW, int C);
/* tiles per frame of the conv launch (0 = tiles may span frames: no fused statistics for that shape) */
int pgt_conv_tiles_per_frame(int Hin, int Win, int Cout, int ksize, int stride, int pad_lo);
/* the same, and 0 when the tile grid does not divide the output frame: a tile past the frame's right or bottom edge
 * adds rows that are not output pixels to its statistics, so the fused statistics are exact only when this is > 0 */
int pgt_conv_tiles_exact(int Hin, int Win, int Cout, int ksize, int stride, int pad_lo);
/* finalize + apply only, with the statistics already produced by the previous conv / linear epilogue
 * (stats: [F, chunks_per_frame, 32, 2], chunks_per_frame = 4 x tiles per frame); saves the statistics pass over the tensor (1/3 of the GroupNorm traffic) */
int pgt_groupnorm_apply_stats(const void* x, int ldx, int F, int HW, int C, const float* gamma, const float* beta,
                              float eps, int apply_silu, void* y, int ldy, const float* stats, int chunks_per_frame,
                              float* ws, void* stream);

/* GroupNorm statistics -> per-(frame, channel) affine terms only: ab[f][0][c] = rstd*gamma, ab[f][1][c] = beta -
 * mean*rstd*gamma (fp32 [F][2][C]), for pgt_conv_gn_bf16.  stats/chunks_per_frame as in pgt_groupnorm_apply_stats, or
 * stats == NULL to compute them from x (ws: pgt_groupnorm_ws_floats floats). */
int pgt_groupnorm_ab(const void* x, int ldx, int F, int HW, int C, const float* gamma, const float* beta, float eps,
                     const float* stats, int chunks_per_frame, float* ws, float* ab, void* stream);
int pgt_groupnorm_silu(const void* x, int ldx, int F, int HW, int C, const float* gamma, const float* beta,
                       float eps, int apply_silu, void* y, int ldy, float* ws, void* stream);

/* ---- LayerNorm over the last dim (eps 1e-5) of a [T, C] matrix; x may be bf16 or fp32.
 * y = LN(x) (bf16); if y2 != NULL also y2 = LN(x) + pos (bf16; pos bf16 [T, ldpos]) — the
 * q = k = LN(x)+pos input of TransformerSALayer (archs/codeformer_arch.py:126-128).
 * Replaces nn.LayerNorm in VSTSREncoderTransformerBlock (modules/rstt_layers.py:298,335),
 * TransformerSALayer norm1/norm2, idx_pred_layer.0. */
int pgt_layernorm(const void* x, int ldx, int x_dtype, int T, int C, const float* gamma, const float* beta,
                  float eps, void* y, int ldy, const void* pos, int ldpos, void* y2, int ldy2, void* stream);

/* ---- LayerNorm fused into the GEMM that consumes it (C = 256, N % 256 == 0):  out[T, N] = LN(x) W^T + bias in ONE kernel —
 * the normalised token matrix never reaches HBM.  W: bf16 [N, ldw] row-major ([out, in]).  Returns PGT_ERR_UNSUPPORTED
 * otherwise.  ln_g == ln_b == NULL: plain normalisation (x - mean) * rstd — the caller has folded gamma / beta into
 * W and bias (W * gamma along the input dim, bias + W beta), which spares the kernel 2 x 256 parameter reads per row.
 * Replaces norm1 + the q / kv projections of VSTSREncoderTransformerBlock / WindowAttention3D
 * (modules/rstt_layers.py:116-132,176-188,326-330). */
int pgt_ln_linear_bf16(const void* x, int ldx, int T, int C, const float* ln_g, const float* ln_b, float eps,
                       const void* W, int ldw, int N, const float* bias, void* out, int ldo, void* stream);

/* ---- fused Swin MLP half-block (C = 256):  out = x + fc2(GELU(fc1(LayerNorm(x)))) in ONE kernel — the hidden tile
 * stays in shared memory / registers, x is read once and out written once.  W1, W2: bf16 [C, C] row-major ([out, in]);
 * gn_stats: optional GroupNorm partials of `out` as in pgt_epilogue.  ln_g == ln_b == NULL: plain normalisation (the
 * caller folded gamma / beta into W1 / b1, as for pgt_ln_linear_bf16).  Returns PGT_ERR_UNSUPPORTED for C != 256.
 * Replaces norm2 + Mlp + residual of VSTSREncoderTransformerBlock (modules/rstt_layers.py:116-132,335-336). */
int pgt_swin_mlp_bf16(const void* x, int ldx, int T, int C, const float* ln_g, const float* ln_b, float eps,
                      const void* W1, const float* b1, const void* W2, const float* b2, void* out, int ldo,
                      float* gn_stats, void* stream);

/* ---- shifted-window spatio-temporal attention core (3 x 4 x 4 windows, N = 48 tokens).
 * qkv: bf16 [F*H*W, 3C] = [q | k | v] per token in natural (frame, y, x) order; the cyclic
 * shift, window partition / reverse and the {0,-100} shift mask are index math inside the
 * kernel; out: bf16 [F*H*W, C] in natural order.  bias_tab: fp32 [heads, 48, 48] (the 245x8
 * relative-position table expanded through relative_position_index at load time).
 * Replaces window_partition/roll/WindowAttention3D core/window_reverse
 * (modules/rstt_layers.py:55-88,213-230,301-329,552-568). */
int pgt_window_attention(const void* qkv, int ldqkv, int clips, int H, int W, int C, int heads, int shift,
                         const float* bias_tab, void* out, int ldo, void* stream);

/* The same core on TMA + wgmma (window_attn_tc.cu): a window's q / k / v rows of a 64-column chunk are one 5-D TMA box
 * of the qkv matrix (wrapped windows of a shifted block: 2 or 4 partial boxes), QK^T and PV run as wgmma with S / P / O
 * in registers, results are stored to the tokens' output rows.  tab: fp16 [4][heads][6][48][8] bias tables
 * (pgtformer_b200/ops.py::window_tables — the relative-position bias in the row order of the four box layouts, times
 * log2 e; the {0,-100} shift mask is not in the table, the kernel adds it in fp32).  mode_n64: for d = 32 run P V with
 * N = 64 instead of a half-atom N = 32 operand view.
 * Returns PGT_ERR_UNSUPPORTED unless heads == 8, d in {32, 64}, C % 128 == 0, shift in {0, 2}. */
int pgt_window_attention_tc(const void* qkv, int ldqkv, int clips, int H, int W, int C, int heads, int shift,
                            const void* tab, void* out, int ldo, int mode_n64, void* stream);

/* ---- generic 3-D shifted-window attention core of the Video-Swin BasicLayer (window3d.cu; modules/swin.py:136-166,
 * 214-250, 309-323; used by TDRQVAE, archs/tdrqvae_arch.py:834-835): window (wd, wh, ww) with wd*wh*ww <= 128, shift
 * (sd, sh, sw), feature map [B, D, H, W] zero-padded to multiples of the window AFTER the projection of the normalised
 * tokens (pad_qkv = the qkv projection of a zero token, i.e. its bias, or NULL for zeros), get_window_size applied
 * here.  qkv bf16 [B*D*H*W, ldqkv] (q | k | v); bias fp32 [heads, N, N] = relative_position_bias_table[
 * relative_position_index[:N, :N]]; out bf16 [B*D*H*W, ldo].  Head dims 16 / 32 / 64. */
int pgt_window3d_attention(const void* qkv, int ldqkv, const void* pad_qkv, int B, int D, int H, int W, int C, int heads,
                           int wd, int wh, int ww, int sd, int sh, int sw, const float* bias, void* out, int ldo,
                           void* stream);

/* ---- global multi-head attention (flash-attention forward, no mask), per clip:
 * q,k,v: bf16 [clips*L, ld*] with head h at columns [h*d, (h+1)*d); out bf16 [clips*L, ldo].
 * Replaces the nn.MultiheadAttention core (archs/codeformer_arch.py:105,129-130); the
 * head-averaged attention weights the reference materialises (need_weights=True) are never
 * consumed (`[0]` at :130) and are not produced.  Head widths 64, 256 and 512; d = 256 / 512 (any L >= 1) is the core
 * of TDRQVAE's dense AttnBlock (archs/tdrqvae_arch.py:151-203: clips = frames, heads = 1, d = C) and needs 16-byte
 * aligned q / k / v / out, else PGT_ERR_UNSUPPORTED. */
int pgt_mha_fwd(const void* q, int ldq, const void* k, int ldk, const void* v, int ldv, int clips, int L,
                int heads, int d, void* out, int ldo, void* stream);

/* ---- codebook ops.
 * pgt_argmax_gather: idx[t] = argmax_k logits[t,k] (first maximum), quant[t,:] = codebook[idx[t],:].
 *   logits fp32 [T, K]; codebook fp32 [K(+1), E]; idx int64 [T]; quant bf16/fp32 [T, ldq].
 *   Replaces logits.argmax(-1) + RQBottleneck.embed_code (archs/pgtformer_arch.py:663-664,
 *   archs/tdcrqvae3_arch.py:354-368).  If idx_in != NULL the argmax is skipped and idx_in is used
 *   (teacher-forced codes).
 * pgt_l2_argmin: idx[t] = argmin_k ||z[t]-e[k]||^2 over the first K codebook rows, lowest index on
 *   ties; z fp32 [T, E] NHWC; also emits quant = e[idx] when quant != NULL.
 *   Replaces VQEmbedding.compute_distances + find_nearest_embedding (archs/tdcrqvae3_arch.py:99-126;
 *   identical copies archs/rqvae_arch.py:218-244, archs/tdrqvae_arch.py:226-251). */
int pgt_argmax_gather(const float* logits, int T, int K, const float* codebook, int E, const int64_t* idx_in,
                      int64_t* idx, void* quant, int ldq, int quant_dtype, void* stream);
int pgt_l2_argmin(const float* z, int T, int E, const float* codebook, int K, int64_t* idx, float* quant,
                  void* stream);
/* The same result on wgmma (l2_argmin_tc.cu): bf16 tensor-core scores of all K codes + a rigorous error window
 * around the approximate minimum; the window's members are re-evaluated exactly (fp32, fp64 when closer than the fp32
 * bound), tokens whose window does not fit go through the exhaustive kernel above — equal to an fp64 argmin with
 * first-index tie-break for every input.
 *   pgt_codebook_pack (load time): cb_bf16 [K, E] bf16 copy, cb_norm [K + 2] fp32 = ||e_k||^2, max||e~||^2, max||e - e~||^2.
 *   workspace: int32 [pgt_l2_argmin_ws_ints(T)] scratch (fallback list + per-token candidate lists).
 *   Returns PGT_ERR_UNSUPPORTED unless K % 256 == 0, E % 128 == 0, E <= 512 (callers then use pgt_l2_argmin). */
int pgt_codebook_pack(const float* codebook, int K, int E, void* cb_bf16, float* cb_norm, void* stream);
int64_t pgt_l2_argmin_ws_ints(int T);
int pgt_l2_argmin_tc(const float* z, int T, int E, const float* codebook, const void* cb_bf16, const float* cb_norm,
                     int K, int64_t* idx, float* quant, int32_t* workspace, void* stream);

/* ---- soft codes of one quantiser depth (RQBottleneck.get_soft_codes, archs/tdcrqvae3_arch.py:429-457).
 * pgt_soft_codes: out[t, k] = softmax_k((2 z[t].e_k - ||e_k||^2) / temp) = softmax_k(-||z[t] - e_k||^2 / temp) over the
 *   first K codebook rows; z fp32 [T, E]; codebook fp32 [K(+1), E]; cb_norm fp32 [>= K] = ||e_k||^2 (the norms
 *   pgt_codebook_pack writes); out fp32 [T, K].  3xTF32 tensor-core dot products (soft_codes.cu), fp32 softmax.
 *   temp must be finite and > 0.  Returns PGT_ERR_UNSUPPORTED unless K % 128 == 0 and E % 32 == 0.
 * pgt_sample_codes: idx[t] = one draw from row t of p fp32 [T, K] (non-negative, any positive sum), Philox keyed by the
 *   DEVICE int64 seed[2]; a zero-probability index is never drawn; a row with no positive entry yields -1.  Replaces
 *   torch.multinomial(soft_code, 1) (:441-444). */
int pgt_soft_codes(const float* z, int T, int E, const float* codebook, const float* cb_norm, int K, float temp,
                   float* out, void* stream);
int pgt_sample_codes(const float* p, int T, int K, const int64_t* seed, int64_t* idx, void* stream);
/* The same two with a row pitch (elements, ldo / ldp >= K, ldo % 4 == 0): at quantiser depth D, depth d writes and
 * reads the K-slice d of a contiguous [T, D, K] soft-code tensor (ldo = D * K), as RQBottleneck.get_soft_codes
 * concatenates them (:429-457).  pgt_soft_codes / pgt_sample_codes are the pitch = K case. */
int pgt_soft_codes_ld(const float* z, int T, int E, const float* codebook, const float* cb_norm, int K, float temp,
                      float* out, int ldo, void* stream);
int pgt_sample_codes_ld(const float* p, int T, int K, int ldp, const int64_t* seed, int64_t* idx, void* stream);

/* ---- residual quantisation over D code levels (rq.cu; RQBottleneck.quantize / embed_code / embed_partial_code /
 * embed_code_with_depth, archs/tdcrqvae3_arch.py:294-426).  Level d's code is pgt_l2_argmin_tc of the level's residual.
 * pgt_rq_residual: one quantiser step after that argmin: e = codebook_d[idx[t]] (codebook_d fp32 [K(+1), E], the
 *   depth's own codebook), r_out = r_in - e (skipped when r_out == NULL, i.e. at the last depth), agg = first ? e :
 *   agg + e (skipped when agg == NULL: the soft-code loop needs only the residual).  fp32, elementwise, one rounding per operation (no FMA): bit-identical to the reference's
 *   residual_feature.sub_(quant) / aggregated_quants.add_(quant) (:319-324) wherever the codes agree.  r_in, r_out,
 *   agg fp32 [T, E] contiguous; E % 4 == 0; r_in may equal r_out.
 * pgt_rq_embed: out[t] = sum over d = d0 .. d1 of codebooks[d * cb_stride + idx[t * ldi + d * ldd] * E], accumulated in
 *   depth order in fp32 from the first term, written fp32 or bf16 (out_dtype) with row pitch ldo.  codebooks: the
 *   stacked [D, K + 1, E] fp32 codebooks (cb_stride = (K + 1) * E) or one shared codebook (cb_stride = 0); idx int64
 *   with token pitch ldi and depth pitch ldd ([T, D] codes: ldi = D, ldd = 1; depth-major [D, T]: ldi = 1, ldd = T).
 *   d0 = 0, d1 = D - 1 is embed_code (:355-368), d1 = j the 'add' mode of embed_partial_code, d0 = d1 = j its
 *   'select' mode and one slice of embed_code_with_depth (:371-426).  Index n_embed reads the padding row; no range
 *   check is made on the device. */
int pgt_rq_residual(const float* r_in, float* r_out, const int64_t* idx, int T, int E, const float* codebook_d,
                    float* agg, int first, void* stream);
int pgt_rq_embed(const int64_t* idx, long long ldi, long long ldd, int T, int d0, int d1, const float* codebooks,
                 long long cb_stride, int E, void* out, int ldo, int out_dtype, void* stream);

/* ---- VectorQuantizer.forward of VQGAN / CodeFormer (vq.cu; archs/vqgan_arch.py:42-84) after the nearest-code argmin:
 * z fp32 [T, E] token rows (T = b * HW, rows of image i are i*HW .. i*HW + HW - 1), codebook fp32 [K, E], idx int64 [T].
 * Per token: zq_nchw fp32 [b, E, HW] and / or zq_bf16 [T, E] = z + (e - z) (fp32, one rounding per operation);
 * min_enc fp32 [T, K] one-hot rows; scores fp32 [T] = exp(-d / 10), d = |z|^2 + |e|^2 - 2 z.e in fp64 rounded to fp32;
 * usage int32 [K] += code counts.  Any of these may be NULL.  hist int32 [K] must be zero on entry (it receives this
 * call's counts); ws: pgt_vq_stats_ws_doubles(T, E) doubles.  scalars fp32 [3] = (loss = m + beta m with
 * m = mean((e - z)^2), perplexity of this call's counts, mean_distance = mean of d over all [T, K] pairs, in closed
 * form), finished on the device; the scalars are deterministic.  E % 32 == 0, E <= 512, K % 4 == 0. */
long long pgt_vq_stats_ws_doubles(int T, int E);
int pgt_vq_stats(const float* z, int T, int E, int HW, const float* codebook, int K, const int64_t* idx, float beta,
                 float* zq_nchw, void* zq_bf16, float* min_enc, float* scores, int* usage, int* hist, double* ws,
                 float* scalars, void* stream);

/* ---- AdaIN: y = (q - mean_q)/std_q * std_l + mean_l per (frame, channel) over HW, unbiased
 * variance + eps.  q: bf16/fp32 [F, HW, ldq]; l (style) bf16 [F, HW, ldl]; y bf16.
 * Replaces adaptive_instance_normalization (archs/codeformer_arch.py:15-46). */
int pgt_adain(const void* q, int ldq, int q_dtype, const void* l, int ldl, int F, int HW, int C, float eps,
              void* y, int ldy, void* stream);

/* ---- face-parsing branch (BiSeNet / ResNet18, archs/pgtformer_arch.py:34-397); its other convolutions run on
 * pgt_conv_bf16 / pgt_conv_up2x_bf16 / pgt_linear_bf16 with eval-mode BatchNorm folded into weights and bias.
 * (the 7x7 stem is pgt_conv_rgb_bf16)
 * pgt_maxpool3x3s2: MaxPool2d(3, 2, 1) (:84,:94)        pgt_global_avgpool: F.avg_pool2d(x, x.size()[2:]) -> bf16 [F,C]
 * pgt_channel_affine: y = x * (scale[f,c] (+1)) + addv[f,c] + addm — ARM / FFM re-weighting (:203, :236-245, :331-333)
 * pgt_assemble_cond: bilinear(align_corners) resize of heads 0,1 to (h16,w16) + head 2, concatenated into the
 *   64-wide (57 used) conditioning map (:375-379). */
int pgt_maxpool3x3s2(const void* x, int ldx, int F, int H, int W, int C, void* y, int ldy, void* stream);
int pgt_global_avgpool(const void* x, int ldx, int F, int HW, int C, void* y, int ldy, void* stream);
int pgt_channel_affine(const void* x, int ldx, int F, int HW, int C, const void* scale, int lds, int plus_one,
                       const void* addv, int ldv, const void* addm, int ldm, void* y, int ldy, void* stream);
int pgt_assemble_cond(const void* o0, int ld0, const void* o1, int ld1, const void* o2, int ld2, int F, int h8, int w8,
                      int h16, int w16, int ncls, void* cond, int ldc, void* stream);

/* ---- layout / elementwise helpers on NHWC bf16 */
/* strided copy of a [T, C] block (concat building: archs/pgtformer_arch.py:467-475) */
int pgt_copy2d(const void* x, int ldx, int T, int C, void* y, int ldy, void* stream);
/* temporal regroup for the SFT block's cross-frame 1x1 mixers (archs/pgtformer_arch.py:467-472):
 * dir 0: x [clips,3,P,C] -> y [clips,P,3C] (channel = frame*C + c); dir 1: the inverse. */
int pgt_regroup_frames(const void* x, int ldx, int clips, int P, int C, void* y, int ldy, int dir, void* stream);
/* fp32 NCHW -> bf16 NHWC (optionally (x-mean[c])/std[c]); bf16 NHWC -> fp32 NCHW / NHWC */
int pgt_nchw_f32_to_nhwc_bf16(const float* x, int F, int C, int HW, const float* mean, const float* stdv, void* y,
                              int ldy, void* stream);
int pgt_nhwc_bf16_to_f32(const void* x, int ldx, int F, int HW, int C, float* y, int to_nchw, void* stream);

/* ---- streaming video front / back end (SURVEY 8f #1): the two conversions of the reference's frame loop and the
 * frame gather that lets per-frame work be computed once per distinct frame.
 *   pgt_u8hwc_to_f32nchw: rgb24 [F, H, W, 3] -> fp32 [F, 3, H, W], y = (float)(v / 255.0) exactly as numpy forms it
 *     (rgbnp2tensor, inference.py:6-10).
 *   pgt_f32nchw_to_u8hwc: frames first, first+step, ... (n of them) of fp32 [*, 3, H, W] -> rgb24 [n, H, W, 3] with
 *     uint8(clamp(x, 0, 1) * 255) (apply_net_to_frames, inference.py:15-19); first = 1, step = 3 selects the middle
 *     frame of every clip.
 *   pgt_gather_frames: y[f] = x[idx[f]] for frames of frame_bytes bytes (multiple of 16); idx: DEVICE int32 [n]. */
int pgt_u8hwc_to_f32nchw(const void* x_u8, int F, int H, int W, float* y, void* stream);
int pgt_f32nchw_to_u8hwc(const float* x, int first, int step, int n, int H, int W, void* y_u8, void* stream);
int pgt_gather_frames(const void* x, long long frame_bytes, const int* idx_dev, int n, void* y, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PGT_B200_H_ */
