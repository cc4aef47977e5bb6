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
"""
import numpy as np
import torch

from . import ops


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
    def __init__(self, model, w=1.0, adain=True, clips_per_batch=16, reuse_frames=True):
        self.model = model
        self.w = float(w)
        self.adain = bool(adain)
        self.clips_per_batch = int(clips_per_batch)
        self.reuse_frames = bool(reuse_frames)

    # ------------------------------------------------------------------ one batch of windows on the device
    def _enqueue(self, frames_u8_dev, local_windows):
        """frames_u8_dev: uint8 [Fd,H,W,3] on the device (distinct frames lo..hi); local_windows: [(a,b,c)] indices
        into it.  Returns uint8 [count,H,W,3] on the device (the restored middle frames)."""
        eng = self.model.engine()
        Fd, H, W, _ = frames_u8_dev.shape
        with torch.cuda.device(eng.dev):
            return self._enqueue_on_device(eng, frames_u8_dev, local_windows, Fd, H, W)

    def _enqueue_on_device(self, eng, frames_u8_dev, local_windows, Fd, H, W):
        x = ops.u8hwc_to_f32nchw(frames_u8_dev, torch.empty(Fd, 3, H, W, dtype=torch.float32, device=frames_u8_dev.device))
        idx = torch.tensor([j for win in local_windows for j in win], dtype=torch.int32).to(x.device, non_blocking=True)
        if self.reuse_frames:
            out = eng.forward(x, w=self.w, adain=self.adain, frame_index=idx)[0]
        else:
            xc = ops.gather_frames(x, idx, torch.empty(idx.numel(), 3, H, W, dtype=torch.float32, device=x.device))
            out = eng.forward(xc, w=self.w, adain=self.adain)[0]
        n = len(local_windows)
        return ops.f32nchw_to_u8hwc(out, torch.empty(n, H, W, 3, dtype=torch.uint8, device=x.device), first=1, step=3)

    def _run_batch(self, frames_u8, local_windows):
        """Host uint8 [Fd,H,W,3] + window index triples -> host uint8 [count,H,W,3] (synchronous; `stream()` uses it)."""
        dev = self.model.engine().dev
        d = torch.from_numpy(np.ascontiguousarray(frames_u8)).pin_memory().to(dev, non_blocking=True)
        return self._enqueue(d, local_windows).cpu().numpy()

    # ------------------------------------------------------------------ whole sequence in memory
    @torch.no_grad()
    def restore(self, frames_u8):
        """frames_u8: uint8 [N,H,W,3] (numpy or torch, host).  Returns numpy uint8 [N,H,W,3]."""
        frames = torch.as_tensor(np.ascontiguousarray(frames_u8)) if not torch.is_tensor(frames_u8) else frames_u8
        if frames.dtype != torch.uint8 or frames.dim() != 4 or frames.shape[-1] != 3:
            raise ValueError('expected rgb24 frames [N,H,W,3] uint8, got %s %s' % (tuple(frames.shape), frames.dtype))
        n = frames.shape[0]
        if n == 0:
            return np.zeros((0,) + tuple(frames.shape[1:]), np.uint8)
        out = torch.empty(frames.shape, dtype=torch.uint8).pin_memory()
        dev = self.model.engine().dev
        main = torch.cuda.current_stream(dev)
        copy = torch.cuda.Stream(dev)
        wins = window_indices(n)
        staged = None                                  # frames of the NEXT batch already on their way
        plan = plan_batches(n, self.clips_per_batch)

        def stage(b):
            first, cnt, lo, hi = plan[b]
            host = frames[lo:hi + 1].contiguous()
            host = host if host.is_pinned() else host.pin_memory()
            with torch.cuda.stream(copy):
                d = host.to(dev, non_blocking=True)
                ev = torch.cuda.Event()
                ev.record(copy)
            return d, ev, host

        staged = stage(0)
        for b, (first, cnt, lo, hi) in enumerate(plan):
            d, ev, _keep = staged
            staged = stage(b + 1) if b + 1 < len(plan) else None     # H2D of the next batch overlaps this compute
            main.wait_event(ev)
            res = self._enqueue(d, [tuple(j - lo for j in wins[i]) for i in range(first, first + cnt)])
            done = torch.cuda.Event()
            done.record(main)
            with torch.cuda.stream(copy):                            # D2H overlaps the next batch's compute
                copy.wait_event(done)
                out[first:first + cnt].copy_(res, non_blocking=True)
            res.record_stream(copy)                                  # the allocator keeps `res` until the copy has run
            d.record_stream(main)
        copy.synchronize()
        main.synchronize()
        return out.numpy()

    # ------------------------------------------------------------------ iterator in, iterator out (bounded memory)
    @torch.no_grad()
    def stream(self, frame_iter):
        """Yields restored rgb24 frames for an iterator of rgb24 frames [H,W,3] uint8, `clips_per_batch` windows per
        launch; the last frame of a batch needs its successor, so output lags the input by one batch."""
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
            res = self._run_batch(np.stack(buf[lo - base:hi - base + 1]), local)
            for k in range(cnt):
                yield res[k]
            emitted += cnt
            drop = max(emitted - 1, 0) - base             # frames before emitted-1 are never needed again
            if drop > 0:
                del buf[:drop]
                base += drop
