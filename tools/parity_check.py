"""Parity of the CUDA forward against the committed golden vectors (outputs OF THE UNMODIFIED REFERENCE, minted by
oracle/make_golden.py) — shared by tests/, __graft_entry__.smoke() and bench.py's `parity` key.
Reads only tests/golden/*; neither the reference nor the oracle is needed at run time.  Large reference tensors are
stored as fixed strided samples (make_golden.sample_into); `sample` takes the same elements of our output.

Numbers reported per fixture (all against the reference's fp32 CPU forward on the same seeded input):
  lq_rel, logits_rel   max|d| / max|ref| of lq_feat and of the sampled logit rows
  code_agree           fraction of tokens whose argmax code equals the reference's
  code_agree_confident the same over tokens whose reference top-1 / top-2 logit margin exceeds 3 * the measured
                       max logit error (a flip there would be a real error, not bf16 noise on a near-tie)
  psnr_tf              PSNR of the middle output frame with the reference's codes teacher-forced (decoder parity)
  psnr_free            PSNR of the free-running middle output frame (code flips change whole 16x16 patches)
"""
import math
import os

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
COMPACT = {512: 'pgtformer_ref_b1_512_seed3_compact.pt', 1024: 'pgtformer_ref_b1_1024_seed4_compact.pt'}
DEMO = 'demo_video_first8.npz'


def golden_input(seed, b, H):
    """Bit-identical to oracle.make_golden.golden_input (kept here so that bench / smoke do not import oracle/)."""
    g = torch.Generator().manual_seed(seed)
    return torch.rand(b * 3, 3, H, H, generator=g)


def sample(t, g, key):
    """The elements of t that fixture g keeps for `key` (t must have the reference tensor's full shape)."""
    assert tuple(t.shape) == tuple(g[key + '_shape']), (tuple(t.shape), g[key + '_shape'])
    return t.float().cpu().reshape(-1)[::g[key + '_stride']]


def psnr(a, b, peak=1.0):
    mse = (a.double() - b.double()).pow(2).mean().item()
    return 99.0 if mse == 0 else 10.0 * math.log10(peak * peak / mse)


def load_compact(size):
    return torch.load(os.path.join(GOLDEN, COMPACT[size]), map_location='cpu')


@torch.no_grad()
def check_compact(model, size, dev='cuda'):
    """Runs `model` on the fixture's input and returns the parity numbers (floats) described in the module docstring."""
    g = load_compact(size)
    x = golden_input(g['seed'], g['b'], g['H']).to(dev)
    out, logits, lq = model(x, w=1, adain=True)
    Fr = x.shape[0]
    hh = size // 16
    lo = logits.reshape(Fr * hh * hh, -1).float().cpu()
    lq = lq.float().cpu()
    st = g['lq_stride']
    ref_lq = g['lq_feat'].float()
    lq_rel = ((sample(lq[:, ::st, ::st], g, 'lq_feat') - ref_lq).abs().max() / g['lq_absmax']).item()
    rows = g['logit_rows_idx'].long()
    logit_err = (lo[rows] - g['logit_rows']).abs().max().item()
    logits_rel = logit_err / g['logits_absmax']
    ref_codes = g['codes'].long().reshape(-1)
    codes = lo.argmax(-1)
    agree = (codes == ref_codes).float().mean().item()
    margin = (g['top2'][..., 0] - g['top2'][..., 1]).reshape(-1)
    conf = margin > 3.0 * logit_err
    agree_conf = (codes[conf] == ref_codes[conf]).float().mean().item() if conf.any() else 1.0
    ref_mid = g['out_mid'].float()
    out_tf = model(x, w=1, adain=True, force_codes=ref_codes.view(Fr, hh, hh, 1).to(dev))[0]
    res = {'size': size, 'lq_rel': lq_rel, 'logits_rel': logits_rel, 'logit_abs_err': logit_err, 'code_agree': agree,
           'code_agree_confident': agree_conf, 'confident_frac': conf.float().mean().item(),
           'psnr_tf': psnr(sample(out_tf[1::3], g, 'out_mid'), ref_mid), 'psnr_free': psnr(sample(out[1::3], g, 'out_mid'), ref_mid),
           'out_tf_rel': ((sample(out_tf[1::3], g, 'out_mid') - ref_mid).abs().max() / g['out_absmax']).item()}
    if hasattr(model, 'forward_vq'):
        vq = model.forward_vq(x, code_only=True)[2].reshape(-1).cpu()
        res['vq_code_agree'] = (vq == g['vq_codes'].long().reshape(-1)).float().mean().item()
    return res


def load_demo():
    import numpy as np
    d = np.load(os.path.join(GOLDEN, DEMO))
    return d['frames'], d['restored']


@torch.no_grad()
def check_demo_video(model, clips_per_batch=8):
    """`inference.py`'s frame loop on the first 8 frames of assets/inputdemovideo.mp4 (downscaled to 128^2) through
    VideoRestorer vs the reference's uint8 output for the same frames.  With the synthetic (untrained) checkpoint there is no ground truth:
    `psnr_vs_reference` is the direct PSNR between the two restorations, `psnr_delta_db` the difference of their PSNRs
    against the input frames (the reading of "PSNR delta vs ref" that carries over to trained weights, where the
    common target is the clean video)."""
    import numpy as np
    from pgtformer_b200.video import VideoRestorer
    frames, ref = load_demo()
    got = VideoRestorer(model, w=1.0, adain=True, clips_per_batch=clips_per_batch).restore(frames)
    f = torch.from_numpy(frames.astype(np.float32))
    a, b = torch.from_numpy(got.astype(np.float32)), torch.from_numpy(ref.astype(np.float32))
    p_got, p_ref = psnr(a, f, 255.0), psnr(b, f, 255.0)
    return {'frames': int(frames.shape[0]), 'psnr_vs_reference': psnr(a, b, 255.0), 'psnr_ours_vs_input': p_got,
            'psnr_ref_vs_input': p_ref, 'psnr_delta_db': p_got - p_ref,
            'byte_equal_frac': float((got == ref).mean()), 'mean_abs_diff_u8': float(np.abs(got.astype(np.int32) - ref.astype(np.int32)).mean())}
