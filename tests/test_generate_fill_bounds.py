"""gnnb_radius_fill with offsets that do not belong to its arguments (csrc/knn.cu).

The C ABI lets a caller pass any offsets to the fill.  Offsets from a count with another r, or corrupted ones, must make
the call fail with GNNB_EINVAL (ValueError here) and must not write outside each row's own range nor past `capacity`:
the entries behind the buffer are checked to be untouched.
"""
import ctypes as C

import numpy as np
import pytest
import torch

GUARD = 4096
SENTINEL = -7


def _count(lib, x, r):
    n, d = x.shape
    off = torch.empty(n + 1, dtype=torch.int64, device="cuda")
    tot = C.c_int64(0)
    lib.check(lib.lib.gnnb_radius_count(x.data_ptr(), n, d, None, 1, float(r), 0, off.data_ptr(), C.byref(tot),
                                        torch.cuda.current_stream().cuda_stream))
    return off, int(tot.value)


def _fill(lib, x, r, off, capacity):
    """fill into a buffer of `capacity` entries followed by GUARD sentinel entries; returns the whole buffer"""
    n, d = x.shape
    buf = torch.full((capacity + GUARD,), SENTINEL, dtype=torch.int32, device="cuda")
    err = None
    try:
        lib.check(lib.lib.gnnb_radius_fill(x.data_ptr(), n, d, None, 1, float(r), 0, off.data_ptr(), buf.data_ptr(),
                                           capacity, torch.cuda.current_stream().cuda_stream))
    except ValueError as e:
        err = e
    return buf, err


@pytest.mark.gpu
def test_fill_with_foreign_offsets_stays_in_bounds():
    from gnnb200 import _lib
    rng = np.random.default_rng(0)
    x = torch.as_tensor(rng.random((3000, 3)).astype(np.float32)).cuda()
    off, tot = _count(_lib, x, 0.1)
    buf, err = _fill(_lib, x, 0.1, off, tot)                 # matching offsets: fine, every slot written
    assert err is None and int((buf[:tot] == SENTINEL).sum()) == 0 and bool((buf[tot:] == SENTINEL).all())

    buf, err = _fill(_lib, x, 0.2, off, tot)                 # more hits per row than the offsets hold
    assert err is not None
    assert bool((buf[tot:] == SENTINEL).all())
    rows = off.cpu().numpy()
    for part in np.split(buf[:tot].cpu().numpy(), rows[1:-1]):   # each row holds the first of its own hits only
        assert (np.diff(part) > 0).all() and (part >= 0).all()

    buf, err = _fill(_lib, x, 0.05, off, tot)                # fewer hits than the offsets hold
    assert err is not None and bool((buf[tot:] == SENTINEL).all())

    bad = off.clone()
    bad[1000:] += 10 ** 9                                    # corrupted offsets pointing far past the buffer
    bad[-1] = off[-1]                                        # ... with a total that passes the capacity check
    buf, err = _fill(_lib, x, 0.1, bad, tot)
    assert err is not None and bool((buf[tot:] == SENTINEL).all())
