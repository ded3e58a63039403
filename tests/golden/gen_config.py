"""Golden of the shipped model config: the parts of the merged `bevformer_base_occ.py` (with its `_base_` files) that the
drop-in surface reads (plugin, model, dist_params), as `Config.fromfile` returns them, stored as JSON so the drop-in tests can
build the detector from it without the reference tree.

    OCC_REFERENCE_ROOT=<reference tree> python tests/golden/gen_config.py
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from occnet_b200.mmcv_shim import Config  # noqa: E402

REL = 'projects/configs/bevformer/bevformer_base_occ.py'
KEYS = ('plugin', 'plugin_dir', 'model', 'dist_params')
OUT = os.path.join(ROOT, 'tests', 'golden', 'ref_config_base_occ.json')


def main():
    cfg = Config.fromfile(os.path.join(os.environ['OCC_REFERENCE_ROOT'], REL))
    d = {k: cfg._cfg_dict[k] for k in KEYS}
    with open(OUT, 'w') as f:                      # one line per top-level key
        f.write('{\n' + ',\n'.join(json.dumps(k) + ':' + json.dumps(d[k], sort_keys=True, separators=(',', ':'))
                                    for k in sorted(d)) + '\n}\n')
    print('wrote', OUT, os.path.getsize(OUT), 'bytes')


if __name__ == '__main__':
    main()
