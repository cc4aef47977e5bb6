"""TEST INFRASTRUCTURE — CPU restatement of the reference's streaming frame loop, used only by tests/ as the checker
for pgtformer_b200/video.py.  Not a product path.

Restates the reference's `inference.py`:
  * `rgbnp2tensor` (:6-10)            rgb24 frames -> float32 [t,3,h,w] via numpy's double division
  * `apply_net_to_frames` (:12-19)    model(window)[0][1] -> clamp -> * 255 -> uint8 (truncation)
  * `process_video_ffmpeg` (:37-76)   the three-frame buffer: first frame duplicated, one window per new frame, last
                                      frame duplicated for the final window
Parity is pinned by construction (the loop is restated line by line, the arithmetic is numpy's own); the model inside
the window is whatever callable the test passes.
"""
import numpy as np


def rgbnp2tensor(window):
    """inference.py:6-10 without the .cuda(): uint8 frames -> float32 [t,3,h,w].  The division happens in float64
    (uint8 array / python float) and is rounded to float32 afterwards — the device kernel must match that rounding."""
    stacked = np.stack([np.asarray(f) for f in window])               # [t,h,w,c] uint8
    unit = (stacked / 255.0).astype(np.float32)
    return np.ascontiguousarray(np.moveaxis(unit, 3, 1))


def tensor2rgb(restored_middle):
    """inference.py:15-18: restored_middle float32 [3,h,w] -> uint8 [h,w,3]."""
    unit = np.clip(np.asarray(restored_middle, np.float32), 0, 1)      # torch.clamp(., 0, 1)
    scaled = np.moveaxis(unit, 0, 2) * 255                              # float32 * python int stays float32
    return scaled.astype(np.uint8)                                      # truncation, values are in [0, 255]


def restore_frames(frames, apply_window):
    """inference.py:37-76 over any iterable of frames.  apply_window(list of 3 frames) -> restored middle frame.

    The reference keeps a three-slot buffer: it is primed with the first frame twice (:43-46), every further frame is
    pushed and, the buffer being full, one window is restored and the oldest slot dropped (:49-70); when the input ends
    with two slots filled, the newest frame is pushed once more and the last window restored (:72-76)."""
    import collections
    restored = []
    slots = collections.deque()
    src = iter(frames)
    head = next(src, None)
    if head is None:
        return restored
    slots.extend((head, head))
    for nxt in src:
        slots.append(nxt)
        if len(slots) == 3:
            restored.append(apply_window(list(slots)))
            slots.popleft()
    if len(slots) == 2:
        slots.append(slots[-1])
        restored.append(apply_window(list(slots)))
    return restored
