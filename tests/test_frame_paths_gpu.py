"""Every frame path of the engine keeps its output bits and its launch schedule: self mode with and without bev_embed, an
explicit prev_bev (map and angle), the video history, channels-last bf16 input and taps, in fp32 and bf16 with and without
tensor cores.  tests/golden/gen_frame_paths.py wrote tests/golden/frame_paths.json; each frame must reproduce its output
digests, launches_per_frame and the per-category launch counts of profile_read."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def check_frame_paths(name):
    sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden'))
    import gen_frame_paths as G
    want = json.load(open(os.path.join(ROOT, 'tests', 'golden', 'frame_paths.json')))[name]
    kw, precision, tc = next((kw, p, tc) for n, kw, p, tc in G.CASES if n == name)
    got = G.run_case(kw, precision, tc)
    assert sorted(got) == sorted(want), name
    for frame in want:
        assert got[frame] == want[frame], f'{name} / {frame}'


@pytest.mark.parametrize('name', ['small6_fp32', 'small6_fp32_tc', 'small6_bf16', 'small6_bf16_tc'])
def test_small6_frame_paths(name):
    check_frame_paths(name)


def test_full_size_frame_paths():
    """in a child process: a device fault in the full-size run must not poison this session's context"""
    code = "import sys; sys.path.insert(0, 'tests'); import test_frame_paths_gpu as t; t.check_frame_paths('full6_bf16_tc'); print('OK')"
    r = subprocess.run([sys.executable, '-c', code], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and 'OK' in r.stdout, f'child failed ({r.returncode}):\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}'
