"""CUDA-graph capture of the rasterizer (torch.cuda.graph): capacity and the sticky status word.

Under `torch.cuda.is_current_stream_capturing()` diff_gauss calls the capture-safe entry points
(sfgs_rasterize_forward_graph / sfgs_rasterize_backward_graph, include/sfgs.h): no host wait, no copy back, the camera
intrinsics optionally in device memory.  Two things the eager forward learns on the host are then handled here:

* the binning capacity, which the eager forward sizes from a running estimate and re-runs when it was too small.  A
  captured forward runs once at a fixed capacity: the one set by `with capacity(n):` around the capture, or else the
  library's estimate for (device, P, width, height) from earlier eager calls plus the eager forward's own margin;
* the frame's error flags (binning overflow, a failed `prefiltered` test, a non-finite subpixel offset), which a
  replay ORs into one device word per device.  `status(device)` reads and clears it; `check(device)` raises
  `SfgsError` naming the bits.  A replay whose frame overflowed has garbage images and zero blend gradients, so check
  before the optimizer step and run that step again eagerly (or re-capture with a larger capacity).

The word is created the first time `status`, `check` or `status_word` runs outside a capture; call one of them once on
each device before its first capture.
"""
from __future__ import annotations

import contextlib
import threading

import torch

from . import native as N

OVERFLOW = 1     # SFGS_STATUS_OVERFLOW
PREFILTER = 2    # SFGS_STATUS_PREFILTER
OFFSET = 4       # SFGS_STATUS_OFFSET
BIT_NAMES = {
    OVERFLOW: "binning overflow (the frame has more tile instances than the captured capacity)",
    PREFILTER: "prefiltered was set but a Gaussian failed the frustum test",
    OFFSET: "a subpixel offset is NaN or Inf",
}

_local = threading.local()
_words: dict = {}


def _index(device) -> int:
    d = torch.device(device) if not isinstance(device, torch.device) else device
    if d.type != "cuda":
        raise ValueError(f"expected a CUDA device, got {d}")
    return d.index if d.index is not None else torch.cuda.current_device()


@contextlib.contextmanager
def capacity(n: int):
    """Binning capacity (tile instances) of every rasterizer forward captured inside the block."""
    n = int(n)
    if n <= 0:
        raise ValueError("capacity must be > 0")
    stack = _local.__dict__.setdefault("stack", [])
    stack.append(n)
    try:
        yield n
    finally:
        stack.pop()


def estimate(device, P: int, width: int, height: int):
    """The eager forward's running instance-count estimate for (device, P, width, height), or None (read-only)."""
    v = int(N.lib().sfgs_capacity_estimate(_index(device), int(P), int(width), int(height)))
    return None if v < 0 else v


def resolve_capacity(device, P: int, width: int, height: int) -> int:
    """The capacity a forward captured now is given: the innermost `capacity(n)`, else the estimate plus the eager
    forward's margin (estimate + estimate / 4 + 4096)."""
    stack = getattr(_local, "stack", None)
    if stack:
        return stack[-1]
    est = estimate(device, P, width, height)
    if est is None:
        raise N.SfgsError(f"no binning capacity for a captured rasterizer forward (P={int(P)}, {int(width)}x{int(height)} "
                          f"on cuda:{_index(device)}): run one eager step first or set a capacity with "
                          "`with sfgs.graphs.capacity(n):` around the capture")
    return est + est // 4 + 4096


def status_word(device) -> torch.Tensor:
    """The device's sticky status word (int32 [1]); created, zeroed, outside a capture only."""
    i = _index(device)
    w = _words.get(i)
    if w is None:
        if torch.cuda.is_current_stream_capturing():
            raise N.SfgsError(f"the rasterizer's status word of cuda:{i} does not exist yet: call "
                              "sfgs.graphs.status(device) once before capturing")
        w = torch.zeros(1, dtype=torch.int32, device=torch.device("cuda", i))
        _words[i] = w
    return w


def status(device) -> int:
    """Read and clear the status word (bits OVERFLOW, PREFILTER, OFFSET); synchronises with the device."""
    w = status_word(device)
    v = int(w.item())
    if v:
        w.zero_()
    return v


def describe(bits: int) -> str:
    return "; ".join(name for b, name in BIT_NAMES.items() if bits & b)


def check(device) -> None:
    """Raise SfgsError if a replay since the last read set any status bit (the word is cleared either way)."""
    v = status(device)
    if v:
        raise N.SfgsError(f"rasterizer graph replay on cuda:{_index(device)} failed (status {v:#x}): {describe(v)}")
