"""Context = device + stream (replaces runtime::buffer::vulkan::Instance,
src/runtime/buffer/vulkan/mod.rs:45-153)."""
from __future__ import annotations

import ctypes as C

from . import _lib
from ._lib import Handle, lib, check


class Context(Handle):
    """One CUDA device + the stream all work of this context is ordered on.

    With ``stream=None`` and torch importable, the context adopts torch's *current* stream of
    that device, so torch tensors, ``torch.cuda.Event`` timing and NCCL collectives issued by
    ``torch.distributed`` are ordered with our kernels without extra synchronisation.
    """
    _destroy = lib.b2s_ctx_destroy

    def __init__(self, device: int = 0, stream: int | None = None, own_stream: bool = False):
        self.device = int(device)
        if stream is None and not own_stream:
            import torch
            if not torch.cuda.is_available():
                raise RuntimeError("futuresdr_b200 needs a CUDA device (no CPU fallback)")
            stream = torch.cuda.current_stream(self.device).cuda_stream
        h = C.c_void_p()
        if own_stream:
            check(lib.b2s_ctx_create(self.device, C.byref(h)))
        else:
            # NB: torch's default stream has handle 0 (the legacy default stream) -- still "on stream"
            check(lib.b2s_ctx_create_on_stream(self.device, C.c_void_p(stream or 0), C.byref(h)))
        self._h = h

    @property
    def handle(self):
        return self._h

    def sync(self):
        check(lib.b2s_ctx_sync(self._h), self._h)

    @property
    def sm_count(self) -> int:
        return lib.b2s_ctx_sm_count(self._h)

    @property
    def launch_count(self) -> int:
        return int(lib.b2s_ctx_launch_count(self._h))

    @property
    def bytes_held(self) -> int:
        """Device + pinned bytes held by the objects created on this context."""
        return int(lib.b2s_ctx_bytes_held(self._h))

    @property
    def stream(self) -> int:
        return lib.b2s_ctx_stream(self._h) or 0


_default: dict[int, Context] = {}


def default_context(device: int | None = None) -> Context:
    """Process-wide context on torch's current device/stream (created on first use)."""
    import torch
    if device is None:
        device = torch.cuda.current_device()
    ctx = _default.get(device)
    if ctx is None:
        ctx = _default[device] = Context(device)
    return ctx
