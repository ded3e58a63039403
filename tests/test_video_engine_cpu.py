"""Argument checks of the video entry points (occb200_engine_set_history, _forward_video, _submit_host_video) through the C
ABI.  They run before any CUDA call, so they need no GPU: return code 1 (an argument check, not 2, a CUDA error) and a
message.  The checks that need a live engine (history not enabled, busy slot, host map out of range) are in
test_video_engine_gpu.py."""
import ctypes

import pytest

FAKE = 1 << 12                       # never dereferenced: every call below is rejected before it reads a buffer


def _call(lib_built, name, *args):
    from occnet_b200 import _lib
    lib = _lib.load()
    rc = getattr(lib, 'occb200_' + name)(*args)
    return rc, lib.occb200_last_error().decode()


def _feats(n=4):
    return (ctypes.c_void_p * 4)(*([FAKE] * n + [None] * (4 - n)))


def test_null_engine_is_rejected(lib_built):
    rc, err = _call(lib_built, 'engine_set_history', None, 1)
    assert rc == 1 and 'null engine' in err
    rc, err = _call(lib_built, 'engine_forward_video', None, _feats(), None, 0, None, None, FAKE, None, None, None)
    assert rc == 1 and 'null engine' in err
    rc, err = _call(lib_built, 'engine_submit_host_video', None, 0, _feats(), None, 0, FAKE, FAKE, None)
    assert rc == 1 and 'null engine' in err


def test_null_pointers_are_rejected(lib_built):
    rc, err = _call(lib_built, 'engine_forward_video', None, None, None, 0, None, None, FAKE, None, None, None)
    assert rc == 1 and 'null pointer' in err
    for feats, occ, flow in ((None, FAKE, FAKE), (_feats(), None, FAKE), (_feats(), FAKE, None)):
        rc, err = _call(lib_built, 'engine_submit_host_video', None, 1, feats, None, 0, occ, flow, None)
        assert rc == 1 and 'null pointer' in err, (feats, occ, flow)


@pytest.mark.parametrize('slot', [-1, 2, 7])
def test_bad_slot_is_rejected(slot, lib_built):
    rc, err = _call(lib_built, 'engine_submit_host_video', None, slot, _feats(), None, 0, FAKE, FAKE, None)
    assert rc == 1 and 'slot' in err
