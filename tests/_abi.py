"""Sentinel-padded device buffers for the GPU tests that call the C ABI through ``_lib.call``, and bitwise comparison of
their outputs.

An output buffer holds the elements a call may write plus a tail prefilled with a sentinel of its dtype; ``take``
checks that the tail survived the call before it hands the elements back, so a write past the end fails the test
instead of landing in someone else's memory unnoticed."""
import numpy as np
import torch

SENTINEL = -1234.5      # float32, float64
SENTINEL_INT = -7       # int32, int64
SENTINEL_U8 = 0xA5
TAIL_ROWS = 128         # a write past N inside the last 128-row tile lands in the tail
TAIL_MIN = 257          # and never fewer elements than this, whatever the row width


def sentinel(dtype):
    return SENTINEL_U8 if dtype == torch.uint8 else SENTINEL if dtype.is_floating_point else SENTINEL_INT


def _shape(shape):
    return tuple(int(s) for s in shape) if isinstance(shape, (tuple, list, torch.Size)) else (int(shape),)


def padded(shape, dtype=torch.float32):
    """A flat CUDA buffer of prod(shape) elements followed by a tail of max(128 rows, 257 elements), all sentinel."""
    shape = _shape(shape)
    tail = max(TAIL_ROWS * int(np.prod(shape[1:])), TAIL_MIN)
    return torch.full((int(np.prod(shape)) + tail,), sentinel(dtype), dtype=dtype, device="cuda")


def take(buf, shape, what):
    """Asserts that nothing was written past the first prod(shape) elements of ``buf`` and returns those on the host,
    reshaped."""
    shape = _shape(shape)
    n = int(np.prod(shape))
    bad = int((buf[n:] != sentinel(buf.dtype)).sum())
    assert bad == 0, "%s: %d values written past its %d elements" % (what, bad, n)
    return buf[:n].reshape(shape).cpu()


def bits(t):
    """The bytes of a tensor (NaNs compare by bit pattern), or a host value as is."""
    if not torch.is_tensor(t):
        return t
    t = t.detach().contiguous().reshape(-1)
    return t.to(torch.uint8) if t.dtype == torch.bool else t.view(torch.uint8)


def same(a, b):
    """Bit-identical tensors, or equal host values."""
    a, b = bits(a), bits(b)
    return torch.equal(a, b) if torch.is_tensor(a) else a == b


def snap(out):
    """A copy of every output of a call once the device is done with it."""
    torch.cuda.synchronize()
    return {k: v.detach().clone() if torch.is_tensor(v) else v for k, v in out.items()}


def rows(t, N):
    """Rows [0, N) of ``t`` as a fresh contiguous float32 CUDA buffer of at least one row, so that N = 0 still passes a
    valid pointer."""
    buf = torch.zeros(max(N, 1), *t.shape[1:], device="cuda")
    buf[:N] = t[:N].cuda()
    return buf
