"""Writes tests/golden/jpeg/*.jpg (small files from OpenCV's writer) and jpeg_sha256.json, the SHA-256 of each file's
cv2.imdecode(IMREAD_UNCHANGED) pixels: the decoder's identity stays pinned if the OpenCV version changes.

    python tests/golden/gen_jpeg.py
"""
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import jpeg_decode as J  # noqa: E402

CASES = {  # name: (content, h, w, quality, sampling, restart, optimize)
    'noise_q95_420_rst0_std': ('noise', 48, 64, 95, '420', 0, False),
    'camera_q75_420_rst1_opt': ('camera', 33, 47, 75, '420', 1, True),
    'bars_q5_444_rst7_std': ('bars', 17, 9, 5, '444', 7, False),
    'flat_q100_444_row_opt': ('flat', 8, 8, 100, '444', 'row', True),
    'noise_q50_420_row_std': ('noise', 1, 1, 50, '420', 'row', False),
}

if __name__ == '__main__':
    os.makedirs(os.path.join(HERE, 'jpeg'), exist_ok=True)
    sums = {}
    for i, (name, (kind, h, w, q, s, r, o)) in enumerate(CASES.items()):
        data = J.encode(J.make_image(kind, h, w, seed=100 + i), q, s, r, o)
        with open(os.path.join(HERE, 'jpeg', name + '.jpg'), 'wb') as f:
            f.write(data)
        sums[name] = hashlib.sha256(J.cv2_decode(data).tobytes()).hexdigest()
    with open(os.path.join(HERE, 'jpeg_sha256.json'), 'w') as f:
        json.dump(sums, f, indent=1, sort_keys=True)
