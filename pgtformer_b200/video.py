"""Streaming video restoration around the model — the GPU counterpart of the reference's frame loop
(`inference.py:21-82` `process_video_ffmpeg` + `apply_net_to_frames :12-19` + `rgbnp2tensor :6-10`).

The reference restores frame i from the window (f[i-1], f[i], f[i+1]) — the first and the last frame are duplicated
at the ends — one window per model call, and keeps `clamp(out[0][1], 0, 1) * 255` as uint8.  Here:

* many windows go through the model per launch (`clips_per_batch`);
* every frame belongs to three consecutive windows, but BiSeNet and the attention-free encoder levels look at one
  frame at a time: with `reuse_frames` they run once per DISTINCT frame of the batch and the results are gathered into
  clip order (`Engine.forward(frame_index=...)`), bit-identical to the per-window computation;
* uint8 <-> float conversion happens on the device with numpy's rounding, frames travel as rgb24 through pinned
  buffers, and the host<->device copies of neighbouring batches overlap the compute on a second stream.

The ffmpeg pipes themselves stay in the caller's script (SURVEY section 7): `stream()` takes any iterator of rgb24
frames and yields rgb24 frames, which is exactly what the reference's pipe loop reads and writes.

`LiveRestorer` is the same loop for a source that delivers frames one at a time: each push returns the previous frame,
each frame's per-frame work runs once into a device ring, and every step can replay from a CUDA graph.  `LivePool` runs
many such streams on one model, batching the new frames and the windows of every stream that pushes into one step;
`LiveRestorer` is a pool of one.
"""
import math

import numpy as np
import torch

from . import degrade, metrics, ops


def window_indices(n):
    """Frame indices of the window that restores frame i, for i in range(n) — the reference's buffer logic
    (`inference.py:41-76`): (0, 0, 1), (0, 1, 2), ..., (n-2, n-1, n-1); a single frame gives (0, 0, 0)."""
    return [(max(i - 1, 0), i, min(i + 1, n - 1)) for i in range(n)]


def plan_batches(n, clips_per_batch):
    """[(first window, window count, lo, hi)]: windows first..first+count-1 need the distinct frames lo..hi."""
    out = []
    for first in range(0, n, clips_per_batch):
        cnt = min(clips_per_batch, n - first)
        out.append((first, cnt, max(first - 1, 0), min(first + cnt, n - 1)))
    return out


class VideoRestorer:
    """restore() and stream() take size = (H, W), multiples of 64: frames of any size are then restored at H x W, each
    upsampled on the device as the reference's test set feeds its low-resolution frames to the model (bilinear,
    align_corners=True; ops.u8hwc_resize_to_f32nchw); the pinned host buffers and the host-to-device copies carry the
    source frames, and outputs are rgb24 at H x W.  size is checked when the call is made, before any device work.

    restore(), evaluate() and stream() take downscale = s, 0 < s < 1: the frames are then ground truth, degraded on the
    device as the reference's test set builds its `lr` input (basicsr's antialiased bicubic imresize by s of v / 255.0,
    kept fp32 and unclamped, then bilinear to H x W; pgtformer_b200.degrade), and restored at size, or at the frames'
    own size (multiples of 64) when size is None.  Only the ground-truth bytes cross to the device.  The `lr` protocol
    on 512^2 ground truth is VideoRestorer(model).evaluate(gt, gt, downscale=0.25)."""

    def __init__(self, model, w=1.0, adain=True, clips_per_batch=16, reuse_frames=True, cuda_graph=False):
        """cuda_graph: replay each batch from a CUDA graph (Engine.graphed, one per batch shape), which removes the
        host cost of its launches; the bytes written are the eager ones."""
        self.model = model
        self.w = float(w)
        self.adain = bool(adain)
        self.clips_per_batch = int(clips_per_batch)
        self.reuse_frames = bool(reuse_frames)
        self.cuda_graph = bool(cuda_graph)

    # ------------------------------------------------------------------ one batch of windows on the device
    def _enqueue(self, frames_u8_dev, local_windows, size=None, gt=None, downscale=None):
        """frames_u8_dev: uint8 [Fd,H,W,3] on the device (distinct frames lo..hi); local_windows: [(a,b,c)] indices
        into it.  Returns uint8 [count,H,W,3] on the device (the restored middle frames; with cuda_graph, the graph's
        static output, to be consumed before the next batch); with size, [count,*size,3].  With gt (their ground
        truth, uint8 [count,*,3] on the device): (restored, sse, per-channel ssim) of Engine.restore_and_score.
        downscale (with size): the frames are ground truth, degraded as the `lr` protocol does."""
        eng = self.model.engine()
        idx = torch.tensor([j for win in local_windows for j in win], dtype=torch.int32).to(eng.dev, non_blocking=True)
        kw = dict(w=self.w, adain=self.adain, reuse_frames=self.reuse_frames, size=size)
        if downscale is not None:
            kw['downscale'] = downscale
        if gt is not None:
            if self.cuda_graph:
                return eng.graphed(eng.restore_and_score, (frames_u8_dev, idx, gt), **kw)
            return eng.restore_and_score(frames_u8_dev, idx, gt, **kw)
        if self.cuda_graph:
            return eng.graphed(eng.restore_windows, (frames_u8_dev, idx), **kw)
        return eng.restore_windows(frames_u8_dev, idx, **kw)

    def _run_batch(self, frames_u8, local_windows, size=None, downscale=None):
        """Host uint8 [Fd,H,W,3] + window index triples -> host uint8 [count,H,W,3] (synchronous; `stream()` uses it)."""
        dev = self.model.engine().dev
        d = torch.from_numpy(np.ascontiguousarray(frames_u8)).pin_memory().to(dev, non_blocking=True)
        return self._enqueue(d, local_windows, size, downscale=downscale).cpu().numpy()

    # ------------------------------------------------------------------ whole sequence in memory
    def restore(self, frames_u8, size=None, downscale=None):
        """frames_u8: uint8 [N,H,W,3] (numpy or torch, host).  Returns numpy uint8 [N,H,W,3] ([N,*size,3] with
        size).  downscale: the frames are ground truth, degraded by the `lr` protocol first (class docstring)."""
        frames = _check_video(frames_u8)
        size, downscale = _check_downscale(downscale, frames.shape[1:3], _check_size(size))
        return self._restore(frames, size, downscale=downscale)

    def evaluate(self, frames_u8, gt_u8, size=None, downscale=None):
        """restore(frames_u8, size), scored against the ground truth gt_u8 (uint8 [N,*out_size,3], numpy or host
        torch; out_size is size, or the frames' own size) as the reference's test configuration scores it
        (pgtformer_b200.metrics.score).  -> (restored, {'psnr': float64 [N], 'ssim': float64 [N]}), restored exactly
        what restore returns.  Each batch's ground truth is staged with its input frames and the restored batch is
        scored on the device before its copy back; the scores are the same bits with cuda_graph.  Arguments are
        checked before any device work.  downscale: frames_u8 is ground truth, degraded by the `lr` protocol first
        (class docstring), so evaluate(gt, gt, downscale=0.25) is that protocol end to end."""
        frames = _check_video(frames_u8)
        size, downscale = _check_downscale(downscale, frames.shape[1:3], _check_size(size))
        gt = metrics.check_frames(gt_u8, 'gt_u8')
        shape = (frames.shape[0],) + (size or tuple(frames.shape[1:3])) + (3,)
        if gt.is_cuda or tuple(gt.shape) != shape:
            raise ValueError('gt_u8: expected host frames %s, got %s%s'
                             % (shape, tuple(gt.shape), ' on %s' % gt.device if gt.is_cuda else ''))
        out, sse, ssim = self._restore(frames, size, gt, downscale)
        return out, metrics.finish(sse, ssim, shape[1:3])

    @torch.no_grad()
    def _restore(self, frames, size, gt=None, downscale=None):
        """restore() on checked arguments; with gt (host uint8 [N,*out_size,3]): (restored, sse int64 [N], ssim
        float64 [N,3]), each batch scored on the device (Engine.restore_and_score)."""
        n = frames.shape[0]
        shape = (n,) + (size or tuple(frames.shape[1:3])) + (3,)
        if n == 0:
            out = np.zeros(shape, np.uint8)
            return out if gt is None else (out, np.zeros(0, np.int64), np.zeros((0, 3)))
        out = torch.empty(shape, dtype=torch.uint8).pin_memory()
        if gt is not None:
            sse = torch.empty(n, dtype=torch.int64).pin_memory()
            ssim = torch.empty(n, 3, dtype=torch.float64).pin_memory()
        dev = self.model.engine().dev
        main = torch.cuda.current_stream(dev)
        copy = torch.cuda.Stream(dev)
        wins = window_indices(n)
        staged = None                                  # frames of the NEXT batch already on their way
        plan = plan_batches(n, self.clips_per_batch)

        def pinned(t):
            t = t.contiguous()
            return t if t.is_pinned() else t.pin_memory()

        def stage(b):
            first, cnt, lo, hi = plan[b]
            host = pinned(frames[lo:hi + 1])
            host_gt = pinned(gt[first:first + cnt]) if gt is not None else None
            with torch.cuda.stream(copy):
                d = host.to(dev, non_blocking=True)
                gd = host_gt.to(dev, non_blocking=True) if gt is not None else None
                ev = torch.cuda.Event()
                ev.record(copy)
            return d, gd, ev, (host, host_gt)

        staged = stage(0)
        copied = None
        for b, (first, cnt, lo, hi) in enumerate(plan):
            d, gd, ev, _keep = staged
            staged = stage(b + 1) if b + 1 < len(plan) else None     # H2D of the next batch overlaps this compute
            main.wait_event(ev)
            if self.cuda_graph and copied is not None:
                main.wait_event(copied)                              # a replay rewrites the static output being copied
            res = self._enqueue(d, [tuple(j - lo for j in wins[i]) for i in range(first, first + cnt)], size, gd,
                                downscale)
            res, scores = (res, ()) if gd is None else (res[0], res[1:])
            done = torch.cuda.Event()
            done.record(main)
            with torch.cuda.stream(copy):                            # D2H overlaps the next batch's compute
                copy.wait_event(done)
                out[first:first + cnt].copy_(res, non_blocking=True)
                for host, t in zip((sse, ssim) if scores else (), scores):
                    host[first:first + cnt].copy_(t, non_blocking=True)
                copied = torch.cuda.Event()
                copied.record(copy)
            if not self.cuda_graph:
                for t in (res,) + scores:
                    t.record_stream(copy)                            # the allocator keeps `t` until the copy has run
            d.record_stream(main)
            if gd is not None:
                gd.record_stream(main)
        copy.synchronize()
        main.synchronize()
        return out.numpy() if gt is None else (out.numpy(), sse.numpy(), ssim.numpy())

    # ------------------------------------------------------------------ iterator in, iterator out (bounded memory)
    def stream(self, frame_iter, size=None, downscale=None):
        """Yields restored rgb24 frames for an iterator of rgb24 frames [H,W,3] uint8, `clips_per_batch` windows per
        launch; the last frame of a batch needs its successor, so output lags the input by one batch.  downscale: the
        frames are ground truth, degraded by the `lr` protocol first (class docstring); the scale is checked now and
        against the first frame's size before it reaches the device."""
        size = _check_size(size)
        if downscale is not None:
            downscale = degrade.check_scale(downscale)
        return self._stream(frame_iter, size, downscale)

    @torch.no_grad()
    def _stream(self, frame_iter, size, downscale=None):
        if downscale is None:
            run_batch = self._run_batch if size is None else lambda f, wins: self._run_batch(f, wins, size)
        else:
            checked = []                                  # the model size, once the first frame has been seen

            def run_batch(f, wins):
                if not checked:
                    checked.append(_check_downscale(downscale, f.shape[1:3], size)[0])
                return self._run_batch(f, wins, checked[0], downscale)
        buf, base, total_in, emitted = [], 0, 0, 0       # buf[k] is frame base + k
        it = iter(frame_iter)
        ended = False
        while True:
            while not ended and len(buf) - (emitted - base) < self.clips_per_batch + 1:
                try:
                    buf.append(np.asarray(next(it), dtype=np.uint8))
                    total_in += 1
                except StopIteration:
                    ended = True
            avail = total_in - emitted if ended else total_in - emitted - 1     # windows whose successor is known
            if avail <= 0:
                if ended:
                    return
                continue
            cnt = min(avail, self.clips_per_batch)
            n_known = total_in
            lo = max(emitted - 1, 0)
            hi = min(emitted + cnt, n_known - 1)
            local = [(max(i - 1, 0) - lo, i - lo, min(i + 1, n_known - 1) - lo) for i in range(emitted, emitted + cnt)]
            res = run_batch(np.stack(buf[lo - base:hi - base + 1]), local)
            for k in range(cnt):
                yield res[k]
            emitted += cnt
            drop = max(emitted - 1, 0) - base             # frames before emitted-1 are never needed again
            if drop > 0:
                del buf[:drop]
                base += drop


def _check_w(w):
    """A fidelity weight from the caller, as a float: NaN and infinities raise ValueError."""
    w = float(w)
    if not math.isfinite(w):
        raise ValueError('w must be finite, got %r' % (w,))
    return w


def _check_video(frames_u8):
    """A whole video from the caller, rgb24 [N,H,W,3] uint8 (numpy or host torch), as a torch tensor; else ValueError."""
    frames = torch.as_tensor(np.ascontiguousarray(frames_u8)) if not torch.is_tensor(frames_u8) else frames_u8
    if frames.dtype != torch.uint8 or frames.dim() != 4 or frames.shape[-1] != 3:
        raise ValueError('expected rgb24 frames [N,H,W,3] uint8, got %s %s' % (tuple(frames.shape), frames.dtype))
    return frames


def _check_downscale(downscale, hw, size):
    """(model size, scale) for frames of hw = (h, w) degraded by `downscale`: the scale checked against the frames
    (degrade.plan) and the size (already checked) or, when None, the frames' own size, which must be multiples of
    64.  downscale None: (size, None).  Anything else raises ValueError."""
    if downscale is None:
        return size, None
    hw = (int(hw[0]), int(hw[1]))
    degrade.plan(hw, downscale)
    return _check_size(size or hw), degrade.check_scale(downscale)


def _check_size(size):
    """The model size (H, W) a video is restored at, as a tuple of ints (None stays None): multiples of 64, else
    ValueError."""
    if size is None:
        return None
    try:
        H, W = (int(v) for v in size)
    except (TypeError, ValueError):
        raise ValueError('size must be (H, W), got %r' % (size,)) from None
    if H <= 0 or W <= 0 or H % 64 or W % 64:
        raise ValueError('size must be multiples of 64, got %dx%d' % (H, W))
    return H, W


def _check_frame(frame, hw, size=None):
    """A live frame, checked on the host: rgb24 [H,W,3] uint8 (numpy, or a host or CUDA torch tensor) with H and W
    multiples of 64, and of the stream's size hw unless hw is None.  With the model size `size` = (H, W) the frame is
    a source of any h, w >= 1 with h w <= H W (it is staged in a row of H W 3 bytes).  Returns it as a torch tensor or
    a numpy array."""
    t = frame if torch.is_tensor(frame) else np.asarray(frame)
    u8 = t.dtype == (torch.uint8 if torch.is_tensor(t) else np.uint8)
    if not u8 or t.ndim != 3 or t.shape[-1] != 3:
        raise ValueError('expected an rgb24 frame [H,W,3] uint8, got %s %s' % (tuple(t.shape), t.dtype))
    H, W = int(t.shape[0]), int(t.shape[1])
    if size is None and (H % 64 or W % 64 or H == 0 or W == 0):
        raise ValueError('expected H, W multiples of 64, got %dx%d' % (H, W))
    if size is not None and (H == 0 or W == 0 or H * W > size[0] * size[1]):
        raise ValueError('expected a source frame of at most %d pixels (the model size %dx%d), got %dx%d'
                         % ((size[0] * size[1],) + size + (H, W)))
    if hw is not None and (H, W) != hw:
        raise ValueError('frame size changed inside a stream: %dx%d after %dx%d' % ((H, W) + hw))
    return t


class _PoolState:
    """The device state of a LivePool on one engine and frame size: the engine's ring of per-frame results for S
    streams (Engine.live_ring; with feats, the SFT skip tensors too), the rgb24 frames that produced them (u8, the same
    rows: 3 s + j % 3 holds frame j of stream s, and rows 3S .. 4S - 1 stage a step's new frames), the fp32 frames of a
    step, the output frames, the device step inputs, pinned host buffers and, with cuda_graph, the captured steps.

    The step inputs are one int32 buffer, uploaded by one copy: idx[:S] the new frames' slots; idx[S:4S] the
    windows' ring rows, three per window; idx[4S:7S] the fusion weight of each of those frames (fp32 bits) and
    idx[7S:10S] its AdaIN flag.  In a pool of source frames (lr), idx[10S:13S] holds each new frame's (h, w, byte
    offset from staging row 3S): its rgb24 row holds the source frame packed from the row's first byte, and the step
    upsamples it to the model size hw (Engine.pool_step).  A step is (B new frames, Bw windows, the first Bw0 of them
    restored without the SFT fusion): Engine.pool_step runs the new frames and those Bw0 windows, Engine.window_step
    the others with their per-frame weights (all > 0).  With cuda_graph each distinct step is captured once
    (Engine._capture) and replayed after its inputs are copied into idx: every address a step touches is allocated
    here, outside the graphs, so the ring carries from one replay to the next and one graph serves every choice of
    streams and every mix of their settings.  The key is (B, Bw), or (B, Bw, Bw0) when Bw0 > 0; B and Bw are at most
    S, so a pool holds at most (S + 1)^2 (S + 2) / 2 - 1 graphs, and a pool whose streams all take the same path at
    most (S + 1)^2 - 1; a single stream with w > 0 uses (1, 0), (1, 1) and (0, 1).  They all share one memory pool,
    replayed one at a time on one stream, so their scratch costs one step's worth."""

    def __init__(self, eng, S, hw, feats, cuda_graph, lr=False):
        self.eng, self.S, self.hw, self.feats, self.cuda_graph, self.lr = eng, S, hw, feats, cuda_graph, lr
        H, W = hw
        n_idx = 13 * S if lr else 10 * S
        dev = eng.dev
        with torch.cuda.device(dev):
            self.ring = eng.live_ring(H, W, 1.0 if feats else 0.0, S)
            self.u8 = torch.empty(4 * S, H, W, 3, dtype=torch.uint8, device=dev)
            self.x = torch.empty(S, 3, H, W, dtype=torch.float32, device=dev)
            self.out = torch.empty(S, H, W, 3, dtype=torch.uint8, device=dev)
            self.idx = torch.empty(n_idx, dtype=torch.int32, device=dev)
        self.host_in = torch.empty(S, H, W, 3, dtype=torch.uint8).pin_memory()
        self.host_idx = torch.zeros(n_idx, dtype=torch.int32).pin_memory()
        self.host_out = torch.empty(S, H, W, 3, dtype=torch.uint8).pin_memory()
        self.loaded = None                 # event: the host buffers have reached the device and may be overwritten
        self.graphs = {}
        self.pool = None

    def run(self, B, Bw, Bw0=0):
        """The step's device work, with its inputs already in idx."""
        S, n0 = self.S, 3 * Bw0
        rows, flags = self.idx[S:S + 3 * Bw], self.idx[7 * S:7 * S + 3 * Bw]
        kw = {'sizes': self.idx[10 * S:10 * S + 3 * B]} if self.lr and B else {}
        self.eng.pool_step(self.u8, self.x, self.ring, self.idx[:B] if B else None, rows[:n0] if Bw0 else None, 0.0,
                           flags[:n0], self.out[:Bw0], **kw)
        if Bw > Bw0:
            wgt = self.idx[4 * S + n0:4 * S + 3 * Bw].view(torch.float32)
            self.eng.window_step(rows[n0:], wgt, flags[n0:], self.ring, self.out[Bw0:Bw])

    def recompute(self, rows, srcs=None):
        """The per-frame work of the rgb24 frames in u8[rows], into the same ring rows (after new weights); srcs: the
        (h, w) of each row's source frame in a pool of source frames (lr), upsampled again."""
        for k, r in enumerate(rows):
            if self.lr:
                ops.u8hwc_resize_to_f32nchw(self.u8[r:r + 1], self.x[:1], srcs[k])
            else:
                ops.u8hwc_to_f32nchw(self.u8[r:r + 1], self.x[:1])
            self.eng.frame_step(self.x[:1], r, self.ring)

    def step(self, new, wins, conf):
        """new: [(ring slot, frame)] of the new frames; wins: [ring rows (a, b, c)] of the windows to restore; conf:
        [(w, adain)] of each window.  Runs one step on the current stream; returns the restored frames in the order of
        wins, numpy uint8 [H,W,3] each (one synchronisation)."""
        S, B, Bw = self.S, len(new), len(wins)
        order = [k for k in range(Bw) if not conf[k][0] > 0] + [k for k in range(Bw) if conf[k][0] > 0]
        Bw0 = sum(not w > 0 for w, _ in conf)
        if self.loaded is not None:
            self.loaded.synchronize()      # the previous step's uploads (a step without windows does not wait)
        for k, (slot, t) in enumerate(new):
            row, host = self.u8[3 * S + k], self.host_in[k]
            if self.lr:                    # the source frame, packed from the row's first byte
                h, w = int(t.shape[0]), int(t.shape[1])
                row, host = row.view(-1)[:h * w * 3].view(h, w, 3), host.view(-1)[:h * w * 3].view(h, w, 3)
                self.host_idx[10 * S + 3 * k:10 * S + 3 * k + 3] = torch.tensor([h, w, k * self.u8[0].numel()])
            if torch.is_tensor(t) and t.is_cuda:
                row.copy_(t, non_blocking=True)
            else:
                host.numpy()[...] = t.numpy() if torch.is_tensor(t) else t
                row.copy_(host, non_blocking=True)
            self.host_idx[k] = slot
        self.host_idx[S:S + 3 * Bw] = torch.tensor([r for k in order for r in wins[k]], dtype=torch.int32)
        self.host_idx[4 * S:4 * S + 3 * Bw].view(torch.float32)[:] = torch.tensor(
            [max(conf[k][0], 0.0) for k in order for _ in range(3)], dtype=torch.float32)
        self.host_idx[7 * S:7 * S + 3 * Bw] = torch.tensor([int(conf[k][1]) for k in order for _ in range(3)],
                                                           dtype=torch.int32)
        self.idx.copy_(self.host_idx, non_blocking=True)
        self.loaded = torch.cuda.Event()
        self.loaded.record()
        if not self.cuda_graph:
            self.run(B, Bw, Bw0)
        else:
            key = (B, Bw, Bw0) if Bw0 else (B, Bw)
            graph = self.graphs.get(key)
            if graph is None:              # the step's writes are idempotent: its warm-up runs leave the ring as is
                graph = self.graphs[key] = self.eng._capture(lambda: self.run(B, Bw, Bw0), self.pool)[0]
                self.pool = graph.pool() if self.pool is None else self.pool
            graph.replay()
        if Bw == 0:
            return []
        self.host_out[:Bw].copy_(self.out[:Bw], non_blocking=True)
        done = torch.cuda.Event()
        done.record()
        done.synchronize()
        got = self.host_out.numpy()
        back = {k: i for i, k in enumerate(order)}
        return [got[back[k]].copy() for k in range(Bw)]


class LivePool:
    """Restores several live videos on one model, each one frame behind its input, batching every stream's new frame
    into one step: push({a: fa[i+1], b: fb[j+1]}) returns {a: frame i of a, b: frame j of b}, each restored from its
    stream's window of the reference's loop (window_indices), byte for byte what VideoRestorer.restore gives on that
    stream alone.

    Each step runs the per-frame work (BiSeNet, the frame blocks of the encoder) of all its new frames as one batch
    into staging rows on the device, scatters the results into each stream's three ring slots, and restores the
    windows of every stream that has one as one batch.  Streams open, stall (a push may list any subset of the open
    streams) and end independently.  Each stream has its own fidelity weight w and AdaIN switch (open, configure),
    and may change them between any two calls; all share the frame size, which the first frame pushed while the pool
    holds no frames sets.  Frames are rgb24 [H,W,3] uint8 — numpy, a host torch tensor or a CUDA tensor on the model's
    device — with H and W multiples of 64; outputs are numpy uint8.  With cuda_graph each distinct (new frames,
    windows, windows without fusion) count replays from one CUDA graph (_PoolState), so streams that push together
    replay one graph whatever their settings.  The device state belongs to the model's current engine: after
    load_state_dict(), .to() or refresh() the next step rebuilds it, re-running the per-frame work of every open
    stream's frames still in a window, from the rgb24 frames the pool keeps on the device.  It is rebuilt the same way
    the first time an open stream has w > 0 on a ring built without the SFT skip tensors (a pool of w = 0 streams does
    not move them); a ring that has them keeps them until the state is rebuilt for another reason.

    size = (H, W), multiples of 64: streams of low-resolution sources, restored at H x W.  Each new frame is upsampled
    on the device as the reference's test set feeds its low-resolution frames to the model (bilinear,
    align_corners=True; ops.u8hwc_resize_to_f32nchw), and only its source bytes cross to the device.  Each stream's
    source size, any h x w with h w <= H W, is set by its first frame; streams of different source sizes share steps
    and graphs.  Outputs are rgb24 at H x W.

        pool = LivePool(model, max_streams=8)
        a, b = pool.open(), pool.open(w=0.5, adain=False)
        pool.push({a: a0, b: b0})     # {a: None, b: None}
        pool.push({a: a1})            # {a: frame 0 of a}
        pool.configure(a, w=0.0)      # from frame 1 of a on
        pool.push({a: a2, b: b1})     # {a: frame 1 of a, b: frame 0 of b}
        pool.flush(a)                 # frame 2 of a; handle a is freed
    """

    def __init__(self, model, max_streams, w=1.0, adain=True, cuda_graph=True, size=None):
        """w, adain: the settings of streams opened without their own."""
        if int(max_streams) < 1:
            raise ValueError('max_streams must be at least 1, got %r' % (max_streams,))
        self.size = _check_size(size)
        if self.size is not None and int(max_streams) * self.size[0] * self.size[1] * 3 >= 2 ** 31:
            raise ValueError('%d streams of %dx%d frames overflow the int32 staging offsets'
                             % ((int(max_streams),) + self.size))
        self.model = model
        self.max_streams = int(max_streams)
        self.w = _check_w(w)
        self.adain = bool(adain)
        self.cuda_graph = bool(cuda_graph)
        self._streams = {}                 # handle -> [stream index s (ring rows 3s .. 3s + 2), frames pushed]
        self._conf = {}                    # stream index s -> (w, adain) of the stream open there
        self._src = {}                     # stream index s -> (h, w) of its source frames (with size)
        self._handles = 0
        self._hw = None
        self._state = None

    def open(self, w=None, adain=None):
        """A new stream's handle; w and adain default to the pool's."""
        conf = (self.w if w is None else _check_w(w), self.adain if adain is None else bool(adain))
        if len(self._streams) >= self.max_streams:
            raise ValueError('all %d streams of the pool are open' % self.max_streams)
        s = min(set(range(self.max_streams)) - {v[0] for v in self._streams.values()})
        h = self._handles
        self._handles += 1
        self._streams[h] = [s, 0]
        self._conf[s] = conf
        self._src.pop(s, None)
        return h

    def configure(self, handle, w=None, adain=None):
        """Changes an open stream's w and / or adain: every window restored after this call uses them, including
        the frame its next push or flush returns.  A negative w restores as w = 0 does (no fusion), as in the
        reference."""
        s, _ = self._stream(handle)
        cw, ca = self._conf[s]
        self._conf[s] = (cw if w is None else _check_w(w), ca if adain is None else bool(adain))

    def close(self, handle):
        """Frees a stream's handle without restoring its last frame."""
        self._stream(handle)
        del self._streams[handle]

    def _stream(self, handle):
        try:
            return self._streams[handle]
        except (KeyError, TypeError):
            raise ValueError('unknown or closed stream handle %r' % (handle,)) from None

    def _holds_frames(self):
        return any(n for _, n in self._streams.values())

    # ------------------------------------------------------------------ schedule (host only)
    @torch.no_grad()
    def push(self, frames):
        """frames: {handle: the stream's next frame} (or (handle, frame) pairs) for any subset of the open streams.
        Returns {handle: its stream's previous frame restored, or None for its first frame}."""
        items = list(frames.items()) if hasattr(frames, 'items') else list(frames)
        hw = self._hw if self._holds_frames() else None
        checked, dev = {}, None
        for h, f in items:
            s, n = self._stream(h)
            if h in checked:
                raise ValueError('stream handle %r listed twice' % (h,))
            if self.size is None:
                t = checked[h] = _check_frame(f, hw)
                hw = (int(t.shape[0]), int(t.shape[1]))
            else:                          # each stream keeps the source size of its first frame
                t = checked[h] = _check_frame(f, self._src[s] if n else None, self.size)
            if torch.is_tensor(t) and t.is_cuda:
                dev = dev or next(self.model.parameters()).device
                if t.device != dev:
                    raise ValueError('frame on %s, model on %s' % (t.device, dev))
        if not checked:
            return {}
        new, wins, order = [], [], []
        for h, t in checked.items():
            s, n = self._streams[h]
            new.append((3 * s + n % 3, t))
            if n > 0:
                wins.append(tuple(3 * s + j % 3 for j in (max(n - 2, 0), n - 1, n)))
                order.append(h)
        hw = hw or self.size
        got = self._step(hw, new, wins)
        self._hw = hw
        for h, t in checked.items():
            self._streams[h][1] += 1
            if self.size is not None:
                self._src[self._streams[h][0]] = (int(t.shape[0]), int(t.shape[1]))
        out = dict.fromkeys(checked)
        out.update(zip(order, got))
        return out

    @torch.no_grad()
    def flush(self, handle):
        """The stream's last frame, restored from (f[n-2], f[n-1], f[n-1]) — (f0, f0, f0) for a single frame; None for
        a stream without frames.  Frees the handle."""
        s, n = self._stream(handle)
        try:
            if n == 0:
                return None
            return self._step(self._hw, [], [tuple(3 * s + j % 3 for j in (max(n - 2, 0), n - 1, n - 1))])[0]
        finally:
            del self._streams[handle]

    # ------------------------------------------------------------------ device
    def _step(self, hw, new, wins):
        """One step on the state of the model's current engine for frames of size hw, each window restored with the
        settings of its stream; a state built mid-stream (new weights or device, or a ring without the SFT skip tensors
        when a stream has w > 0) first recomputes the ring from the rgb24 frames it still holds.  A state with the skip
        tensors keeps them while no stream needs them: dropping them would cost a rebuild and new graph captures at
        every crossing."""
        eng = self.model.engine()
        feats = any(self._conf[s][0] > 0 for s, _ in self._streams.values())
        state = old = self._state
        if old is None or old.eng is not eng or old.hw != hw or (feats and not old.feats):
            self._state = None
            state = _PoolState(eng, self.max_streams, hw, feats, self.cuda_graph, self.size is not None)
            if old is not None and old.hw == hw and self._holds_frames():
                live = [(s, j) for s, n in self._streams.values() for j in range(max(n - 2, 0), n)]
                with torch.cuda.device(eng.dev):
                    state.u8.copy_(old.u8)
                    state.recompute([3 * s + j % 3 for s, j in live], [self._src.get(s) for s, _ in live])
            self._state = state
        with torch.cuda.device(eng.dev):
            return state.step(new, wins, [self._conf[win[0] // 3] for win in wins])


class LiveRestorer:
    """Restores a live video one frame behind its input: push(f[i+1]) returns frame i, restored from the window
    (f[i-1], f[i], f[i+1]) of the reference's loop (window_indices), byte for byte what VideoRestorer.restore gives.

    Each frame's per-frame work (BiSeNet, the frame blocks of the encoder) runs once, when it is pushed, into a ring of
    three slots on the device; each window is gathered from the ring.  Frames are rgb24 [H,W,3] uint8 — numpy, a host
    torch tensor or a CUDA tensor on the model's device — with H and W multiples of 64; outputs are numpy uint8.  With
    cuda_graph every step replays from a CUDA graph.  configure() changes w and adain between any two calls.  It is the
    one stream of a LivePool of one.  The device state belongs to the model's current
    engine: after load_state_dict(), .to() or refresh() the next call rebuilds it, re-running the per-frame work of the
    frames still in the window on the new weights.  size = (H, W): a low-resolution source of any h x w with
    h w <= H W, restored at H x W as LivePool(size=...) does.

        live = LiveRestorer(model)
        live.push(f0)     # None
        live.push(f1)     # frame 0, window (0, 0, 1)
        live.push(f2)     # frame 1, window (0, 1, 2)
        live.flush()      # frame 2, window (1, 2, 2); then ready for a new stream
    """

    def __init__(self, model, w=1.0, adain=True, cuda_graph=True, size=None):
        self.model = model
        self.w = _check_w(w)
        self.adain = bool(adain)
        self.cuda_graph = bool(cuda_graph)
        self._pool = LivePool(model, 1, w=w, adain=adain, cuda_graph=cuda_graph, size=size)
        self.size = self._pool.size
        self._handle = None
        self.reset()

    def configure(self, w=None, adain=None):
        """Changes w and / or adain for every window restored after this call, including the frame the next push or
        flush returns, and for the streams after a reset."""
        w = self.w if w is None else _check_w(w)
        adain = self.adain if adain is None else bool(adain)
        if self._handle is not None:
            self._pool.configure(self._handle, w, adain)
        self.w = self._pool.w = w
        self.adain = self._pool.adain = adain

    def reset(self):
        """Forgets the current stream (its frames); the next push starts a new one, of any frame size."""
        self._n = 0            # frames pushed in this stream
        self._hw = None
        if self._handle is not None:
            self._pool.close(self._handle)
            self._handle = None

    # ------------------------------------------------------------------ schedule (host only)
    @torch.no_grad()
    def push(self, frame):
        """Frame n of the stream in; restored frame n - 1 out (None for n = 0)."""
        t = _check_frame(frame, self._hw, self.size)
        if torch.is_tensor(t) and t.is_cuda and t.device != next(self.model.parameters()).device:
            raise ValueError('frame on %s, model on %s' % (t.device, next(self.model.parameters()).device))
        n = self._n
        new = n % 3
        win = None if n == 0 else (max(n - 2, 0), n - 1, n)
        out = self._step(t, n, new, win)
        self._n, self._hw = n + 1, (int(t.shape[0]), int(t.shape[1]))
        return out

    @torch.no_grad()
    def flush(self):
        """The last frame of the stream, restored from (f[n-2], f[n-1], f[n-1]) — (f0, f0, f0) for a single frame;
        None for an empty stream.  Then ready for a new stream."""
        n = self._n
        try:
            return None if n == 0 else self._step(None, n, None, (max(n - 2, 0), n - 1, n - 1))
        finally:
            self.reset()

    def stream(self, frames):
        """Yields restored frame i as soon as frame i + 1 (or the end of `frames`) is known."""
        self.reset()
        for f in frames:
            out = self.push(f)
            if out is not None:
                yield out
        out = self.flush()
        if out is not None:
            yield out

    # ------------------------------------------------------------------ device
    def _step(self, t, n, new, win):
        """t: frame n (or None at flush) going into ring slot `new`; win: frame indices of the window to restore.  The
        one stream of the pool keeps exactly this schedule."""
        if t is None:
            handle, self._handle = self._handle, None
            return self._pool.flush(handle)
        if self._handle is None:
            self._handle = self._pool.open()
        return self._pool.push({self._handle: t})[self._handle]
