"""TEST INFRASTRUCTURE ONLY — mints tests/golden/* by running the UNMODIFIED reference
(a reference checkout, imported through oracle/reference_loader.py) on seeded inputs with the
deterministic synthetic checkpoint (pgtformer_b200.weights.synth_state_dict, seed 0).

Run where the reference checkout is available (PGT_REFERENCE_ROOT); the tests only read tests/golden/*:
    python -m oracle.make_golden            # 128^2 fixtures
    python -m oracle.make_golden --full     # 512^2 (the reference's native size, NO size patch) and 1024^2 (size patch)
    python -m oracle.make_golden --video    # first 8 frames of assets/inputdemovideo.mp4, downscaled to 128^2, through
                                            # inference.py's loop
    python -m oracle.make_golden --swin     # the Video-Swin BasicLayer of modules/swin.py (TDRQVAE) on stand-in weights
Inputs are not stored: `golden_input(seed, b, H)` regenerates them bit-exactly.

The full-size fixtures are stored compactly (the raw outputs are 50-200 MB): every code index (int16), the top-2
logit values of every token (the margin that decides whether a code flip is a real error), full logit rows for a
seeded sample of tokens, lq_feat as fp16 (at 1024^2: every other token in y and x), the middle output frame as fp16
(that is what `inference.py:15` consumes), the L2-argmin codes of `TDCRQVAE3.get_codes`, and per-tensor max|ref|.
Every fixture stays below 1 MB: large tensors are kept as `t.reshape(-1)[::stride]` with key_shape / key_stride /
key_absmax beside them (`sample_into`), and the tests take the same sample of their own output.
"""
import argparse
import os
import sys
import time

import torch
import yaml

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
OPT = os.path.join(ROOT, 'options', 'release_test_stage_IIII_dont_need_align_version.yml')
DEMO_VIDEO = 'assets/inputdemovideo.mp4'          # relative to the reference root
N_LOGIT_ROWS = 384               # seeded token sample; a compact fixture keeps every LOGIT_ROW_STEP-th of them
LOGIT_ROW_STEP = 4
SMALL_STRIDES = {'out': 2, 'logits': 4, 'lq_feat': 2, 'vq_out': 4}     # x b (clips) at 128^2
COMPACT_STRIDES = {512: (8, 12), 1024: (16, 48)}                       # (lq_feat, out_mid) flat sample strides
DEMO_SIZE = 128


def load_network_g():
    with open(OPT) as f:
        return yaml.safe_load(f)['network_g']


def golden_input(seed, b, H):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(b * 3, 3, H, H, generator=g)


def sampled_rows(T, seed):
    """Token rows whose full logit vectors a compact fixture keeps."""
    g = torch.Generator().manual_seed(1000 + seed)
    return torch.randperm(T, generator=g)[:N_LOGIT_ROWS].sort().values


def sample_into(rec, key, t, stride):
    """rec[key] = the strided flat sample of t, with its full shape, stride and max|t|."""
    rec[key] = t.reshape(-1)[::stride].contiguous()
    rec[key + '_shape'] = tuple(t.shape)
    rec[key + '_stride'] = stride
    rec[key + '_absmax'] = t.abs().max().item()


def small_record(out, logits, lq, vq_out, vq_loss, vq_codes, seed, b, H):
    rec = {'seed': seed, 'b': b, 'H': H, 'w': 1.0, 'adain': True, 'codes': logits.argmax(-1),
           'vq_loss': vq_loss, 'vq_codes': vq_codes}
    for key, t in (('out', out), ('logits', logits), ('lq_feat', lq.contiguous()), ('vq_out', vq_out)):
        sample_into(rec, key, t.float(), SMALL_STRIDES[key] * b)
    return rec


def _reference_model():
    from oracle.reference_loader import build_reference_model
    from pgtformer_b200.spec import build_spec
    from pgtformer_b200.weights import synth_state_dict
    opt = load_network_g()
    arch, spec = build_spec(opt)
    sd = synth_state_dict(spec, 0)
    torch.set_num_threads(os.cpu_count())
    return build_reference_model(opt, sd)


def small():
    from oracle.reference_loader import reference_forward, import_reference, generalise_size
    m = _reference_model()
    ref_mod = import_reference()
    for (seed, b, H) in ((1, 1, 128), (2, 2, 128)):
        x = golden_input(seed, b, H)
        out, logits, lq = reference_forward(m, x, w=1.0, adain=True)
        # the registered TDCRQVAE3.forward (L2-argmin path) on the same module / weights
        vq = []
        with torch.no_grad():
            for i in range(b):
                generalise_size(m, H, H)
                vq.append(ref_mod.TDCRQVAE3.forward(m, x[i * 3:(i + 1) * 3]))
        rec = small_record(out, logits, lq, torch.cat([v[0] for v in vq], 0), torch.stack([v[1] for v in vq]),
                           torch.cat([v[2] for v in vq], 0), seed, b, H)
        path = os.path.join(GOLDEN, 'pgtformer_ref_b%d_%d_seed%d.pt' % (b, H, seed))
        torch.save(rec, path)
        print('wrote', path, {k: tuple(v.shape) for k, v in rec.items() if torch.is_tensor(v)})
    # 64^2, small enough to keep whole
    seed, H = 7, 64
    out, logits, lq = reference_forward(m, golden_input(seed, 1, H), w=1.0, adain=True)
    path = os.path.join(GOLDEN, 'pgtformer_ref_b1_%d_seed%d.pt' % (H, seed))
    torch.save({'seed': seed, 'b': 1, 'H': H, 'w': 1.0, 'adain': True, 'out': out, 'logits': logits,
                'lq_feat': lq.contiguous()}, path)
    print('wrote', path)


def compact_record(out, logits, lq, seed, H, lq_stride):
    Fr = out.shape[0]
    T = logits.numel() // logits.shape[-1]
    lo = logits.reshape(T, -1)
    top2 = lo.topk(2, dim=-1)
    rows = sampled_rows(T, seed)[::LOGIT_ROW_STEP]
    lq_flat, out_flat = COMPACT_STRIDES[H]
    rec = {'seed': seed, 'b': Fr // 3, 'H': H, 'w': 1.0, 'adain': True, 'compact': True,
           'codes': lo.argmax(-1).to(torch.int16).view(Fr, H // 16, H // 16),
           'top2': top2.values.float().view(Fr, H // 16, H // 16, 2).contiguous(),
           'logit_rows_idx': rows.to(torch.int32), 'logit_rows': lo[rows].float().contiguous(),
           'logits_absmax': lo.abs().max().item(), 'lq_stride': lq_stride}
    sample_into(rec, 'lq_feat', lq[:, ::lq_stride, ::lq_stride].to(torch.float16), lq_flat)
    rec['lq_absmax'] = lq.abs().max().item()                  # of the whole tensor, not only the y / x subsample
    sample_into(rec, 'out_mid', out[1::3].to(torch.float16), out_flat)
    rec['out_absmax'] = out.abs().max().item()
    return rec


def full():
    """512^2 through the UNPATCHED reference (its native size); 1024^2 through `generalise_size`."""
    from oracle.reference_loader import generalise_size, import_reference
    ref_mod = import_reference()
    for (seed, H, lq_stride) in ((3, 512, 1), (4, 1024, 2)):
        m = _reference_model()                          # fresh module: the 512^2 run sees no run-time patch at all
        if H != 512:
            generalise_size(m, H, H)
        x = golden_input(seed, 1, H)
        t0 = time.time()
        with torch.no_grad():
            out, logits, lq = m(x, w=1.0, adain=True)
            vq_codes = ref_mod.TDCRQVAE3.get_codes(m, x)
        rec = compact_record(out, logits, lq, seed, H, lq_stride)
        rec['vq_codes'] = vq_codes.to(torch.int16).view(3, H // 16, H // 16)
        rec['patched'] = H != 512
        path = os.path.join(GOLDEN, 'pgtformer_ref_b1_%d_seed%d_compact.pt' % (H, seed))
        torch.save(rec, path)
        print('wrote %s in %.0f s (%.1f MB)' % (path, time.time() - t0, os.path.getsize(path) / 1e6),
              {k: tuple(v.shape) for k, v in rec.items() if torch.is_tensor(v)})


def read_demo_frames(n):
    """First n frames of the reference's demo video as rgb24 (cv2 decodes BGR)."""
    import cv2
    import numpy as np
    from oracle.reference_loader import REFERENCE_ROOT
    cap = cv2.VideoCapture(os.path.join(REFERENCE_ROOT, DEMO_VIDEO))
    frames = []
    while len(frames) < n:
        ok, f = cap.read()
        if not ok:
            break
        frames.append(cv2.cvtColor(f, cv2.COLOR_BGR2RGB))
    cap.release()
    return np.stack(frames)


def video(n=8):
    """`inference.py:12-19,37-76` on the first n frames of assets/inputdemovideo.mp4, downscaled to DEMO_SIZE^2 (area
    filter), with the reference model (CPU): the input frames and the reference's uint8 outputs are stored, so the GPU
    test needs neither the video nor the reference."""
    import cv2
    import numpy as np
    from oracle import video_oracle as VO
    from oracle.reference_loader import generalise_size
    m = _reference_model()
    generalise_size(m, DEMO_SIZE, DEMO_SIZE)
    frames = np.stack([cv2.resize(f, (DEMO_SIZE, DEMO_SIZE), interpolation=cv2.INTER_AREA) for f in read_demo_frames(n)])

    def apply_window(win):                               # apply_net_to_frames without the .cuda()
        x = torch.from_numpy(VO.rgbnp2tensor(win))
        with torch.no_grad():
            mid = m(x, w=1.0)[0][1]                      # adain comes from the yml (True), as in inference.py:15
        return VO.tensor2rgb(mid.numpy())

    t0 = time.time()
    restored = np.stack(VO.restore_frames(list(frames), apply_window))
    path = os.path.join(GOLDEN, 'demo_video_first%d.npz' % n)
    np.savez_compressed(path, frames=frames, restored=restored)
    print('wrote %s in %.0f s (%.1f MB)' % (path, time.time() - t0, os.path.getsize(path) / 1e6), frames.shape, restored.shape)


def swin():
    """The reference's Video-Swin `BasicLayer` (`modules/swin.py:326-405`, imported with the mmcv / basicsr / timm shims)
    on the deterministic stand-in weights of oracle/swin3d_oracle.py: outputs stored as fp16."""
    import importlib.util
    from oracle import swin3d_oracle as S
    from oracle.reference_loader import REFERENCE_ROOT, _ensure_paths
    _ensure_paths()
    spec = importlib.util.spec_from_file_location('_pgt_reference.modules.swin', os.path.join(REFERENCE_ROOT, 'modules', 'swin.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    for name, c in S.SWIN_CASES.items():
        layer = mod.BasicLayer(c['dim'], c['depth'], c['heads'], c['window']).eval()
        layer.load_state_dict(S.synth_state(layer.state_dict(), c['seed']), strict=True)
        x = S.case_input(name)
        with torch.no_grad():
            y = layer(x)
        path = os.path.join(GOLDEN, 'swin3d_%s.pt' % name)
        torch.save({'case': name, 'out': y.to(torch.float16), 'out_absmax': y.abs().max().item()}, path)
        print('wrote', path, tuple(y.shape), '%.1f KB' % (os.path.getsize(path) / 1e3))
    # the reference layer's state dict layout (names, shapes, dtypes) and relative position index, for the drop-in
    ref = mod.BasicLayer(256, 4, 8, (5, 5, 5)).state_dict()
    path = os.path.join(GOLDEN, 'swin3d_state_dict_spec.pt')
    torch.save({'spec': {k: (tuple(v.shape), str(v.dtype)) for k, v in ref.items()},
                'relative_position_index': ref['blocks.0.attn.relative_position_index'].to(torch.int16)}, path)
    print('wrote', path)


if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument('--full', action='store_true')
    ap.add_argument('--video', action='store_true')
    ap.add_argument('--swin', action='store_true')
    a = ap.parse_args()
    if a.full:
        full()
    if a.video:
        video()
    if a.swin:
        swin()
    if not (a.full or a.video or a.swin):
        small()
