"""Mint the fixtures of FQF's fraction loss under tests/golden/fqf_fraction/ from the UNMODIFIED reference
(oracle/ref_loader.py).

    python tests/golden/make_fqf_fraction_golden.py

One ``<case>.npz`` per entry of ``tests.test_fqf_fraction.CASES``: the seeded inputs (``in_*``), the case parameters
(``case``, JSON), the loss (``out_loss``) and d loss / d quantiles for the upstream gradients 1 and 0.37 (``out_grad_u1``,
``out_grad_u037``), computed by ``fqf_calculate_fraction_loss`` (ding/rl_utils/td.py:1466-1513) on the CPU.
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import ref_loader  # noqa: E402
from tests import test_fqf_fraction as ff  # noqa: E402


def main():
    if not ref_loader.available():
        raise SystemExit("the reference is not importable here")
    ref = ref_loader.load()
    os.makedirs(ff.GOLDEN_DIR, exist_ok=True)
    for name, case in sorted(ff.CASES.items()):
        t = ff.make_inputs(case)
        arrays = {'case': np.array(json.dumps(case, sort_keys=True))}
        arrays.update({'in_' + k: v.numpy() for k, v in t.items()})
        for u in ff.UPSTREAM:
            out = ff.run(ref, t, 'cpu', u)
            arrays['out_loss'] = out['loss'].astype(np.float32)
            arrays[ff.grad_key(u)] = out['grad'].astype(np.float32)
        np.savez_compressed(os.path.join(ff.GOLDEN_DIR, name + '.npz'), **arrays)
    print("wrote %d cases to %s" % (len(ff.CASES), ff.GOLDEN_DIR))


if __name__ == '__main__':
    main()
