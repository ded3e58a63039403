"""Writes tests/golden/jpeg_streams_sha256.json: the SHA-256 of cv2.imdecode(IMREAD_UNCHANGED)'s pixels for every case of
tests/golden/jpeg_streams.py, so that a different OpenCV shows up as such and not as a decoder failure.  The files
themselves are regenerated from their seeds, never stored.

    python tests/golden/gen_jpeg_streams.py
"""
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)
import jpeg_streams as S  # noqa: E402
from oracle import jpeg_decode as J  # noqa: E402

if __name__ == '__main__':
    sums = {c['name']: hashlib.sha256(J.cv2_decode(c['data']).tobytes()).hexdigest() for c in S.cases()}
    with open(os.path.join(HERE, 'jpeg_streams_sha256.json'), 'w') as f:
        json.dump(sums, f, indent=1, sort_keys=True)
        f.write('\n')
