"""Shared by gen_fullsize.py (writer) and the tests (readers): which elements of a big tensor a golden file holds."""
import numpy as np

N_TAP, N_OUT = 10000, 100000      # positions drawn per tensor (per-layer taps / outputs)
N1 = 40000                        # positions drawn per output of the one-layer goldens (gen_onelayer.py)


def stride(n):
    """Every stride(n)-th of the n drawn positions is stored: 2500 per tap, 10000 per output, so each file stays < 1 MB."""
    return 4 if n <= N_TAP else -(-n // 10000)


def sub_idx(key, numel, n):
    """Sample positions are a pure function of (tensor name, size): regenerated on the test side, not stored."""
    seed = sum((i + 1) * ord(ch) for i, ch in enumerate(key)) % (2 ** 31)
    idx = np.sort(np.random.RandomState(seed).choice(numel, size=min(n, numel), replace=False)).astype(np.int64)
    return idx[::stride(n)]
