// TORCH_LIBRARY shim over the C ABI (include/pgt_b200.h): `torch.ops.pgt.*` for the hot-path kernels, the PyTorch-side
// binding SURVEY 8(b) sketches next to the ctypes one (pgtformer_b200/_lib.py).  Nothing is computed here: every op
// checks dtypes / devices, takes raw device pointers and the current CUDA stream of the tensor's device, and calls the
// same extern "C" entry point the ctypes binding calls.  Built by pgtformer_b200/build.py into lib/libpgt_torch.so
// (plain g++, links libpgt_b200.so); loaded on demand by pgtformer_b200/torch_ops.py.
#include <ATen/ATen.h>
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/library.h>

#include "../../include/pgt_b200.h"

namespace {

void check(int rc, const char* what) {
  if (rc == PGT_OK) return;
  std::string msg = std::string("libpgt_b200 (") + what + "): " + pgt_strerror(rc);
  if (rc == PGT_ERR_CUDA) msg += std::string(": ") + pgt_last_cuda_error();
  TORCH_CHECK(false, msg);
}

void* stream_of(const at::Tensor& t) { return at::cuda::getCurrentCUDAStream(t.device().index()).stream(); }

int ld(const at::Tensor& t) {           // row pitch (elements) of a channels-last [..., C] tensor / view
  TORCH_CHECK(t.stride(-1) == 1, "expected a channels-last tensor");
  return t.dim() > 1 ? (int)t.stride(-2) : (int)t.size(-1);
}

void window_attention(const at::Tensor& qkv, int64_t clips, int64_t H, int64_t W, int64_t C, int64_t heads, int64_t shift,
                      const at::Tensor& tab16, at::Tensor out) {
  TORCH_CHECK(qkv.is_cuda() && qkv.scalar_type() == at::kBFloat16 && out.scalar_type() == at::kBFloat16 &&
              tab16.scalar_type() == at::kHalf && tab16.is_contiguous(), "window_attention: bf16 qkv / out, fp16 table");
  c10::cuda::CUDAGuard guard(qkv.device());
  check(pgt_window_attention_tc(qkv.data_ptr(), ld(qkv), (int)clips, (int)H, (int)W, (int)C, (int)heads, (int)shift,
                                tab16.data_ptr(), out.data_ptr(), ld(out), stream_of(qkv)), "window_attention");
}

void mha_fwd(const at::Tensor& q, const at::Tensor& k, const at::Tensor& v, int64_t clips, int64_t L, int64_t heads, int64_t d,
             at::Tensor out) {
  TORCH_CHECK(q.is_cuda() && q.scalar_type() == at::kBFloat16 && k.scalar_type() == at::kBFloat16 &&
              v.scalar_type() == at::kBFloat16 && out.scalar_type() == at::kBFloat16, "mha_fwd: bf16 tensors");
  c10::cuda::CUDAGuard guard(q.device());
  check(pgt_mha_fwd(q.data_ptr(), ld(q), k.data_ptr(), ld(k), v.data_ptr(), ld(v), (int)clips, (int)L, (int)heads, (int)d,
                    out.data_ptr(), ld(out), stream_of(q)), "mha_fwd");
}

void argmax_gather(const at::Tensor& logits, const at::Tensor& codebook, at::Tensor idx, at::Tensor quant) {
  TORCH_CHECK(logits.is_cuda() && logits.scalar_type() == at::kFloat && logits.is_contiguous() &&
              codebook.scalar_type() == at::kFloat && idx.scalar_type() == at::kLong, "argmax_gather: fp32 logits / codebook, int64 idx");
  c10::cuda::CUDAGuard guard(logits.device());
  const int qd = quant.scalar_type() == at::kBFloat16 ? PGT_BF16 : PGT_F32;
  check(pgt_argmax_gather(logits.data_ptr<float>(), (int)logits.size(0), (int)logits.size(1), codebook.data_ptr<float>(),
                          (int)codebook.size(1), nullptr, idx.data_ptr<int64_t>(), quant.data_ptr(), ld(quant), qd,
                          stream_of(logits)), "argmax_gather");
}

std::tuple<at::Tensor, at::Tensor> codebook_pack(const at::Tensor& codebook, int64_t K) {
  TORCH_CHECK(codebook.is_cuda() && codebook.scalar_type() == at::kFloat && codebook.is_contiguous() && codebook.size(0) >= K);
  c10::cuda::CUDAGuard guard(codebook.device());
  auto cb16 = at::empty({K, codebook.size(1)}, codebook.options().dtype(at::kBFloat16));
  auto norm = at::empty({K + 2}, codebook.options());
  check(pgt_codebook_pack(codebook.data_ptr<float>(), (int)K, (int)codebook.size(1), cb16.data_ptr(), norm.data_ptr<float>(),
                          stream_of(codebook)), "codebook_pack");
  return std::make_tuple(cb16, norm);
}

void l2_argmin(const at::Tensor& z, const at::Tensor& codebook, const at::Tensor& cb16, const at::Tensor& norm, int64_t K,
               at::Tensor idx, const c10::optional<at::Tensor>& quant) {
  TORCH_CHECK(z.is_cuda() && z.scalar_type() == at::kFloat && z.is_contiguous() && codebook.is_contiguous() &&
              idx.scalar_type() == at::kLong, "l2_argmin: fp32 contiguous z / codebook, int64 idx");
  c10::cuda::CUDAGuard guard(z.device());
  const int T = (int)z.size(0), E = (int)z.size(1);
  auto ws = at::empty({pgt_l2_argmin_ws_ints(T)}, z.options().dtype(at::kInt));
  float* qp = quant.has_value() ? quant->data_ptr<float>() : nullptr;
  int rc = pgt_l2_argmin_tc(z.data_ptr<float>(), T, E, codebook.data_ptr<float>(), cb16.data_ptr(), norm.data_ptr<float>(),
                            (int)K, idx.data_ptr<int64_t>(), qp, ws.data_ptr<int>(), stream_of(z));
  if (rc == PGT_ERR_UNSUPPORTED)
    rc = pgt_l2_argmin(z.data_ptr<float>(), T, E, codebook.data_ptr<float>(), (int)K, idx.data_ptr<int64_t>(), qp, stream_of(z));
  check(rc, "l2_argmin");
}

void l2_argmin_split(const at::Tensor& z, const at::Tensor& codebook, const at::Tensor& cb16, const at::Tensor& norm,
                     int64_t K, int64_t splits, at::Tensor idx, const c10::optional<at::Tensor>& quant) {
  TORCH_CHECK(z.is_cuda() && z.scalar_type() == at::kFloat && z.is_contiguous() && codebook.is_contiguous() &&
              idx.scalar_type() == at::kLong && splits >= 1, "l2_argmin_split: fp32 contiguous z / codebook, int64 idx");
  c10::cuda::CUDAGuard guard(z.device());
  const int T = (int)z.size(0), E = (int)z.size(1);
  auto ws = at::empty({pgt_l2_argmin_split_ws_ints(T, (int)splits)}, z.options().dtype(at::kInt));
  float* qp = quant.has_value() ? quant->data_ptr<float>() : nullptr;
  check(pgt_l2_argmin_tc_split(z.data_ptr<float>(), T, E, codebook.data_ptr<float>(), cb16.data_ptr(),
                               norm.data_ptr<float>(), (int)K, (int)splits, idx.data_ptr<int64_t>(), qp, ws.data_ptr<int>(),
                               stream_of(z)), "l2_argmin_split");
}

void soft_codes(const at::Tensor& z, const at::Tensor& codebook, const at::Tensor& norm, int64_t K, double temp,
                at::Tensor out) {
  TORCH_CHECK(z.is_cuda() && z.scalar_type() == at::kFloat && z.is_contiguous() && codebook.scalar_type() == at::kFloat &&
              codebook.is_contiguous() && norm.scalar_type() == at::kFloat && out.scalar_type() == at::kFloat &&
              out.dim() == 2 && out.stride(1) == 1 && out.size(0) == z.size(0) && out.size(1) == K,
              "soft_codes: fp32 contiguous z [T, E], codebook, norm, row-pitched out [T, K]");
  c10::cuda::CUDAGuard guard(z.device());
  check(pgt_soft_codes(z.data_ptr<float>(), (int)z.size(0), (int)z.size(1), codebook.data_ptr<float>(),
                       norm.data_ptr<float>(), (int)K, (float)temp, out.data_ptr<float>(), (int)out.stride(0),
                       stream_of(z)), "soft_codes");
}

void sample_codes(const at::Tensor& p, const at::Tensor& seed, at::Tensor idx) {
  TORCH_CHECK(p.is_cuda() && p.scalar_type() == at::kFloat && p.dim() == 2 && p.stride(1) == 1 &&
              seed.scalar_type() == at::kLong && seed.numel() == 2 && seed.device() == p.device() &&
              idx.scalar_type() == at::kLong && idx.is_contiguous() && idx.numel() == p.size(0),
              "sample_codes: fp32 row-pitched p [T, K], device int64 seed [2], int64 idx [T]");
  c10::cuda::CUDAGuard guard(p.device());
  check(pgt_sample_codes(p.data_ptr<float>(), (int)p.size(0), (int)p.size(1), (int)p.stride(0), seed.data_ptr<int64_t>(),
                         idx.data_ptr<int64_t>(), stream_of(p)), "sample_codes");
}

void rq_residual(const c10::optional<at::Tensor>& r_in, const c10::optional<at::Tensor>& r_out, const at::Tensor& idx,
                 const at::Tensor& codebook, const c10::optional<at::Tensor>& agg, bool first) {
  TORCH_CHECK(agg.has_value() || r_out.has_value(), "rq_residual: agg or r_out is needed");
  const at::Tensor& ref = agg.has_value() ? *agg : *r_out;
  TORCH_CHECK(ref.is_cuda() && ref.dim() == 2 && codebook.scalar_type() == at::kFloat && codebook.is_contiguous() &&
              codebook.size(1) == ref.size(1) && idx.scalar_type() == at::kLong && idx.is_contiguous() &&
              idx.numel() == ref.size(0), "rq_residual: codebook fp32 [K(+1), E], int64 idx [T]");
  for (const auto* r : {&r_in, &r_out, &agg})
    TORCH_CHECK(!r->has_value() || ((*r)->scalar_type() == at::kFloat && (*r)->is_contiguous() &&
                                    (*r)->sizes() == ref.sizes()), "rq_residual: fp32 contiguous [T, E] tensors");
  c10::cuda::CUDAGuard guard(ref.device());
  auto ptr = [](const c10::optional<at::Tensor>& t) { return t.has_value() ? t->data_ptr<float>() : nullptr; };
  check(pgt_rq_residual(ptr(r_in), ptr(r_out), idx.data_ptr<int64_t>(), (int)ref.size(0), (int)ref.size(1),
                        codebook.data_ptr<float>(), ptr(agg), first ? 1 : 0, stream_of(ref)), "rq_residual");
}

void rq_embed(const at::Tensor& idx, int64_t d0, int64_t d1, const at::Tensor& codebooks, at::Tensor out, int64_t ldi,
              int64_t ldd) {
  TORCH_CHECK(idx.is_cuda() && idx.scalar_type() == at::kLong && idx.is_contiguous() && codebooks.scalar_type() == at::kFloat &&
              codebooks.is_contiguous() && codebooks.dim() == 3 && out.dim() == 2 && out.size(1) == codebooks.size(2) &&
              (out.scalar_type() == at::kFloat || out.scalar_type() == at::kBFloat16) && 0 <= d0 && d0 <= d1 &&
              (codebooks.size(0) == 1 || d1 < codebooks.size(0)) && (out.size(0) - 1) * ldi + d1 * ldd < idx.numel(),
              "rq_embed: int64 codes, fp32 codebooks [D or 1, K + 1, E], fp32 / bf16 out [T, E]");
  c10::cuda::CUDAGuard guard(idx.device());
  const int64_t cb_stride = codebooks.size(0) == 1 ? 0 : codebooks.size(1) * codebooks.size(2);
  check(pgt_rq_embed(idx.data_ptr<int64_t>(), ldi, ldd, (int)out.size(0), (int)d0, (int)d1, codebooks.data_ptr<float>(),
                     cb_stride, (int)out.size(1), out.data_ptr(), ld(out),
                     out.scalar_type() == at::kBFloat16 ? PGT_BF16 : PGT_F32, stream_of(idx)), "rq_embed");
}

void linear(const at::Tensor& a, const at::Tensor& w, const c10::optional<at::Tensor>& bias, int64_t act,
            const c10::optional<at::Tensor>& residual, at::Tensor out) {
  TORCH_CHECK(a.is_cuda() && a.scalar_type() == at::kBFloat16 && w.scalar_type() == at::kBFloat16 && w.stride(1) == 1,
              "linear: bf16 a [M, K], w [N, K]");
  c10::cuda::CUDAGuard guard(a.device());
  pgt_epilogue ep;
  memset(&ep, 0, sizeof(ep));
  ep.bias = bias.has_value() ? bias->data_ptr<float>() : nullptr;
  ep.act = (int)act;
  ep.mode = PGT_EPI_PLAIN;
  if (residual.has_value()) {
    ep.residual = residual->data_ptr();
    ep.ldr = ld(*residual);
    ep.res_dtype = residual->scalar_type() == at::kBFloat16 ? PGT_BF16 : PGT_F32;
  }
  ep.out = out.data_ptr();
  ep.ldo = ld(out);
  ep.out_dtype = out.scalar_type() == at::kBFloat16 ? PGT_BF16 : PGT_F32;
  ep.out_layout = PGT_OUT_NHWC;
  const int64_t M = a.numel() / a.size(-1);
  check(pgt_linear_bf16(a.data_ptr(), ld(a), w.data_ptr(), (int)w.stride(0), (int)M, (int)w.size(0), (int)a.size(-1), &ep,
                        stream_of(a)), "linear");
}

void conv_out_gn_act(const at::Tensor& x, const at::Tensor& ab, const at::Tensor& wp, int64_t cout,
                     const c10::optional<at::Tensor>& bias, bool silu, at::Tensor out) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 4 && x.scalar_type() == at::kBFloat16 && x.stride(3) == 1 &&
              x.stride(1) == x.size(2) * x.stride(2) && (x.size(0) == 1 || x.stride(0) == x.size(1) * x.stride(1)) &&
              ab.scalar_type() == at::kFloat && wp.scalar_type() == at::kBFloat16 && wp.stride(1) == 1 &&
              out.scalar_type() == at::kFloat && out.is_contiguous() && out.dim() == 4 && out.size(0) == x.size(0) &&
              out.size(1) == cout && out.size(2) == x.size(1) && out.size(3) == x.size(2),
              "conv_out_gn_act: bf16 x [F, H, W, 64], fp32 ab [F, 2, 64], bf16 packed wp, fp32 out [F, cout, H, W]");
  TORCH_CHECK(ab.device() == x.device() && wp.device() == x.device() && out.device() == x.device() &&
              (!bias.has_value() || (bias->device() == x.device() && bias->scalar_type() == at::kFloat)),
              "conv_out_gn_act: every tensor on x's device, fp32 bias");
  c10::cuda::CUDAGuard guard(x.device());
  check(pgt_conv_out_gn_act(x.data_ptr(), (int)x.size(0), (int)x.size(1), (int)x.size(2), (int)x.size(3), (int)x.stride(2),
                            ab.data_ptr<float>(), wp.data_ptr(), (int)wp.stride(0), (int)cout,
                            bias.has_value() ? bias->data_ptr<float>() : nullptr, out.data_ptr<float>(), silu ? 1 : 0,
                            stream_of(x)), "conv_out_gn_act");
}

void vq_stats(const at::Tensor& z, const at::Tensor& codebook, const at::Tensor& idx, int64_t HW, double beta,
              at::Tensor scalars, const c10::optional<at::Tensor>& zq_nchw, const c10::optional<at::Tensor>& zq_bf16,
              const c10::optional<at::Tensor>& min_enc, const c10::optional<at::Tensor>& scores,
              const c10::optional<at::Tensor>& usage) {
  TORCH_CHECK(z.is_cuda() && z.dim() == 2 && z.scalar_type() == at::kFloat && z.is_contiguous() &&
              codebook.scalar_type() == at::kFloat && codebook.is_contiguous() && codebook.dim() == 2 &&
              codebook.size(1) == z.size(1) && idx.scalar_type() == at::kLong && idx.is_contiguous() &&
              idx.numel() == z.size(0) && scalars.scalar_type() == at::kFloat && scalars.is_contiguous() &&
              scalars.numel() >= 3, "vq_stats: fp32 z [T, E], codebook [K, E], int64 idx [T], fp32 scalars [3]");
  const int64_t T = z.size(0), E = z.size(1), K = codebook.size(0);
  TORCH_CHECK(codebook.device() == z.device() && idx.device() == z.device() && scalars.device() == z.device(),
              "vq_stats: codebook, idx and scalars must be on z's device");
  auto opt = [&z](const c10::optional<at::Tensor>& t, at::ScalarType dt, int64_t n) -> void* {
    if (!t.has_value()) return nullptr;
    TORCH_CHECK(t->scalar_type() == dt && t->is_contiguous() && t->numel() == n, "vq_stats: optional output dtype / size");
    TORCH_CHECK(t->device() == z.device(), "vq_stats: every output must be on z's device");
    return t->data_ptr();
  };
  void* zn = opt(zq_nchw, at::kFloat, T * E);
  void* zb = opt(zq_bf16, at::kBFloat16, T * E);
  void* me = opt(min_enc, at::kFloat, T * K);
  void* sc = opt(scores, at::kFloat, T);
  void* us = opt(usage, at::kInt, K);
  c10::cuda::CUDAGuard guard(z.device());
  auto hist = at::zeros({K}, z.options().dtype(at::kInt));
  auto ws = at::empty({std::max<int64_t>(pgt_vq_stats_ws_doubles((int)T, (int)E), 1)}, z.options().dtype(at::kDouble));
  check(pgt_vq_stats(z.data_ptr<float>(), (int)T, (int)E, (int)HW, codebook.data_ptr<float>(), (int)K,
                     idx.data_ptr<int64_t>(), (float)beta, static_cast<float*>(zn), zb, static_cast<float*>(me),
                     static_cast<float*>(sc), static_cast<int*>(us), hist.data_ptr<int>(), ws.data_ptr<double>(),
                     scalars.data_ptr<float>(), stream_of(z)), "vq_stats");
}

void adain_frames(const at::Tensor& q, const at::Tensor& style, const at::Tensor& flags, double eps, at::Tensor out) {
  TORCH_CHECK(q.is_cuda() && q.dim() == 3 && (q.scalar_type() == at::kFloat || q.scalar_type() == at::kBFloat16) &&
              style.scalar_type() == at::kBFloat16 && style.sizes() == q.sizes() && out.scalar_type() == at::kBFloat16 &&
              out.sizes() == q.sizes() && flags.scalar_type() == at::kInt && flags.is_contiguous() &&
              flags.numel() == q.size(0), "adain_frames: fp32 / bf16 q [F, HW, C], bf16 style and out, int32 flags [F]");
  TORCH_CHECK(style.device() == q.device() && flags.device() == q.device() && out.device() == q.device(),
              "adain_frames: every tensor on q's device");
  TORCH_CHECK(q.stride(1) == ld(q) && style.stride(1) == ld(style) && out.stride(1) == ld(out),
              "adain_frames: row-pitched [F, HW, C] tensors");
  TORCH_CHECK(q.stride(0) == q.size(1) * ld(q) && style.stride(0) == style.size(1) * ld(style) &&
              out.stride(0) == out.size(1) * ld(out), "adain_frames: frames one after another");
  c10::cuda::CUDAGuard guard(q.device());
  check(pgt_adain_frames(q.data_ptr(), ld(q), q.scalar_type() == at::kBFloat16 ? PGT_BF16 : PGT_F32, style.data_ptr(),
                         ld(style), (int)q.size(0), (int)q.size(1), (int)q.size(2), (float)eps, flags.data_ptr<int32_t>(),
                         out.data_ptr(), ld(out), stream_of(q)), "adain_frames");
}

void u8hwc_resize_to_f32nchw(const at::Tensor& x, int64_t h, int64_t w, const c10::optional<at::Tensor>& sizes,
                             at::Tensor out) {
  TORCH_CHECK(x.is_cuda() && x.scalar_type() == at::kByte && x.is_contiguous() && out.scalar_type() == at::kFloat &&
              out.is_contiguous() && out.dim() == 4 && out.size(1) == 3,
              "u8hwc_resize_to_f32nchw: contiguous uint8 x, contiguous fp32 out [F, 3, H, W]");
  TORCH_CHECK(out.device() == x.device(), "u8hwc_resize_to_f32nchw: x and out on one device");
  const int64_t F = out.size(0);
  const int32_t* sp = nullptr;
  if (sizes.has_value()) {
    TORCH_CHECK(sizes->scalar_type() == at::kInt && sizes->is_contiguous() && sizes->numel() == 3 * F &&
                sizes->device() == x.device(), "u8hwc_resize_to_f32nchw: int32 sizes [F, 3] on x's device");
    sp = sizes->data_ptr<int32_t>();
  } else {
    TORCH_CHECK(x.numel() >= F * h * w * 3, "u8hwc_resize_to_f32nchw: x holds fewer than F h w 3 bytes");
  }
  c10::cuda::CUDAGuard guard(x.device());
  check(pgt_u8hwc_resize_to_f32nchw(x.data_ptr(), (int)F, (int)h, (int)w, sp, (int)out.size(2), (int)out.size(3),
                                    out.data_ptr<float>(), stream_of(x)), "u8hwc_resize_to_f32nchw");
}

void f32nchw_resize_to_f32nchw(const at::Tensor& x, at::Tensor out) {
  TORCH_CHECK(x.is_cuda() && x.scalar_type() == at::kFloat && x.is_contiguous() && x.dim() == 4 && x.size(1) == 3 &&
              out.scalar_type() == at::kFloat && out.is_contiguous() && out.dim() == 4 && out.size(1) == 3 &&
              out.size(0) == x.size(0), "f32nchw_resize_to_f32nchw: contiguous fp32 x [F, 3, h, w], out [F, 3, H, W]");
  TORCH_CHECK(out.device() == x.device(), "f32nchw_resize_to_f32nchw: x and out on one device");
  c10::cuda::CUDAGuard guard(x.device());
  check(pgt_f32nchw_resize_to_f32nchw(x.data_ptr<float>(), (int)x.size(0), (int)x.size(2), (int)x.size(3),
                                      (int)out.size(2), (int)out.size(3), out.data_ptr<float>(), stream_of(x)),
        "f32nchw_resize_to_f32nchw");
}

void imresize_u8hwc_to_f32nchw(const at::Tensor& x, const at::Tensor& wts_h, const at::Tensor& idx_h,
                               const at::Tensor& wts_w, const at::Tensor& idx_w, at::Tensor out) {
  TORCH_CHECK(x.is_cuda() && x.scalar_type() == at::kByte && x.is_contiguous() && x.dim() == 4 && x.size(3) == 3 &&
              out.scalar_type() == at::kFloat && out.is_contiguous() && out.dim() == 4 && out.size(1) == 3 &&
              out.size(0) == x.size(0), "imresize_u8hwc_to_f32nchw: contiguous rgb24 x [F, h, w, 3], fp32 out "
              "[F, 3, oh, ow]");
  for (const at::Tensor* t : {&wts_h, &idx_h, &wts_w, &idx_w})
    TORCH_CHECK(t->is_contiguous() && t->dim() == 2 && t->device() == x.device(),
                "imresize_u8hwc_to_f32nchw: contiguous [out, K] tap tables on x's device");
  TORCH_CHECK(wts_h.scalar_type() == at::kFloat && wts_w.scalar_type() == at::kFloat &&
              idx_h.scalar_type() == at::kInt && idx_w.scalar_type() == at::kInt && wts_h.sizes() == idx_h.sizes() &&
              wts_w.sizes() == idx_w.sizes() && wts_h.size(0) == out.size(2) && wts_w.size(0) == out.size(3),
              "imresize_u8hwc_to_f32nchw: fp32 weights and int32 indices [oh, Kh], [ow, Kw]");
  TORCH_CHECK(out.device() == x.device(), "imresize_u8hwc_to_f32nchw: x and out on one device");
  c10::cuda::CUDAGuard guard(x.device());
  check(pgt_imresize_u8hwc_to_f32nchw(x.data_ptr(), (int)x.size(0), (int)x.size(1), (int)x.size(2),
                                      wts_h.data_ptr<float>(), idx_h.data_ptr<int32_t>(), (int)wts_h.size(1),
                                      (int)out.size(2), wts_w.data_ptr<float>(), idx_w.data_ptr<int32_t>(),
                                      (int)wts_w.size(1), (int)out.size(3), out.data_ptr<float>(), stream_of(x)),
        "imresize_u8hwc_to_f32nchw");
}

void frame_scores(const at::Tensor& a, const at::Tensor& b, at::Tensor sse, at::Tensor ssim) {
  TORCH_CHECK(a.is_cuda() && a.scalar_type() == at::kByte && a.is_contiguous() && a.dim() == 4 && a.size(3) == 3 &&
              b.scalar_type() == at::kByte && b.is_contiguous() && b.sizes() == a.sizes(),
              "frame_scores: contiguous rgb24 frames a, b [F, H, W, 3] uint8 of one shape");
  const int64_t F = a.size(0);
  TORCH_CHECK(sse.scalar_type() == at::kLong && sse.is_contiguous() && sse.numel() == F &&
              ssim.scalar_type() == at::kDouble && ssim.is_contiguous() && ssim.numel() == 3 * F,
              "frame_scores: int64 sse [F], fp64 ssim [F, 3]");
  TORCH_CHECK(b.device() == a.device() && sse.device() == a.device() && ssim.device() == a.device(),
              "frame_scores: every tensor on a's device");
  c10::cuda::CUDAGuard guard(a.device());
  const int H = (int)a.size(1), W = (int)a.size(2);
  auto ws = at::empty({std::max<int64_t>(pgt_frame_scores_ws_doubles((int)F, H, W), 1)}, a.options().dtype(at::kDouble));
  check(pgt_frame_scores(a.data_ptr(), b.data_ptr(), (int)F, H, W, ws.data_ptr<double>(),
                         reinterpret_cast<uint64_t*>(sse.data_ptr<int64_t>()), ssim.data_ptr<double>(), stream_of(a)),
        "frame_scores");
}

}  // namespace

TORCH_LIBRARY(pgt, m) {
  m.def("window_attention(Tensor qkv, int clips, int H, int W, int C, int heads, int shift, Tensor tab16, Tensor(a!) out) -> ()");
  m.def("mha_fwd(Tensor q, Tensor k, Tensor v, int clips, int L, int heads, int d, Tensor(a!) out) -> ()");
  m.def("argmax_gather(Tensor logits, Tensor codebook, Tensor(a!) idx, Tensor(b!) quant) -> ()");
  m.def("codebook_pack(Tensor codebook, int K) -> (Tensor, Tensor)");
  m.def("l2_argmin(Tensor z, Tensor codebook, Tensor cb16, Tensor norm, int K, Tensor(a!) idx, Tensor(b!)? quant) -> ()");
  m.def("l2_argmin_split(Tensor z, Tensor codebook, Tensor cb16, Tensor norm, int K, int splits, Tensor(a!) idx, "
        "Tensor(b!)? quant) -> ()");
  m.def("linear(Tensor a, Tensor w, Tensor? bias, int act, Tensor? residual, Tensor(a!) out) -> ()");
  m.def("soft_codes(Tensor z, Tensor codebook, Tensor norm, int K, float temp, Tensor(a!) out) -> ()");
  m.def("sample_codes(Tensor p, Tensor seed, Tensor(a!) idx) -> ()");
  m.def("rq_residual(Tensor? r_in, Tensor(a!)? r_out, Tensor idx, Tensor codebook, Tensor(b!)? agg, bool first) -> ()");
  m.def("rq_embed(Tensor idx, int d0, int d1, Tensor codebooks, Tensor(a!) out, int ldi, int ldd) -> ()");
  m.def("conv_out_gn_act(Tensor x, Tensor ab, Tensor wp, int cout, Tensor? bias, bool silu, Tensor(a!) out) -> ()");
  m.def("vq_stats(Tensor z, Tensor codebook, Tensor idx, int HW, float beta, Tensor(a!) scalars, Tensor(b!)? zq_nchw, "
        "Tensor(c!)? zq_bf16, Tensor(d!)? min_enc, Tensor(e!)? scores, Tensor(f!)? usage) -> ()");
  m.def("adain_frames(Tensor q, Tensor style, Tensor flags, float eps, Tensor(a!) out) -> ()");
  m.def("u8hwc_resize_to_f32nchw(Tensor x, int h, int w, Tensor? sizes, Tensor(a!) out) -> ()");
  m.def("frame_scores(Tensor a, Tensor b, Tensor(a!) sse, Tensor(b!) ssim) -> ()");
  m.def("f32nchw_resize_to_f32nchw(Tensor x, Tensor(a!) out) -> ()");
  m.def("imresize_u8hwc_to_f32nchw(Tensor x, Tensor wts_h, Tensor idx_h, Tensor wts_w, Tensor idx_w, Tensor(a!) out) "
        "-> ()");
}

TORCH_LIBRARY_IMPL(pgt, CUDA, m) {
  m.impl("window_attention", window_attention);
  m.impl("mha_fwd", mha_fwd);
  m.impl("argmax_gather", argmax_gather);
  m.impl("codebook_pack", codebook_pack);
  m.impl("l2_argmin", l2_argmin);
  m.impl("l2_argmin_split", l2_argmin_split);
  m.impl("linear", linear);
  m.impl("soft_codes", soft_codes);
  m.impl("sample_codes", sample_codes);
  m.impl("rq_residual", rq_residual);
  m.impl("rq_embed", rq_embed);
  m.impl("conv_out_gn_act", conv_out_gn_act);
  m.impl("vq_stats", vq_stats);
  m.impl("adain_frames", adain_frames);
  m.impl("u8hwc_resize_to_f32nchw", u8hwc_resize_to_f32nchw);
  m.impl("frame_scores", frame_scores);
  m.impl("f32nchw_resize_to_f32nchw", f32nchw_resize_to_f32nchw);
  m.impl("imresize_u8hwc_to_f32nchw", imresize_u8hwc_to_f32nchw);
}
