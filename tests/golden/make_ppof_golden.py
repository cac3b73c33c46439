"""Mint the fixtures of PPOFPolicy's advantage recompute under tests/golden/ppof/ from the UNMODIFIED reference
(oracle/ref_loader.py).

    python tests/golden/make_ppof_golden.py

One ``<case>.npz`` per entry of ``tests.test_ppof.CASES``: the seeded inputs (``in_*``; an input that is None is absent),
the case parameters (``case``, JSON), and adv / value / return_ (``out_adv``, ``out_value``, ``out_return``) plus, for
'baseline', (mean, population variance, count) of return_ (``out_stats``), computed on the CPU by ding/policy/ppof.py:160-210
as restated around the live reference functions in tests/ppof_oracle.py.
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import ref_loader  # noqa: E402
from tests import test_ppof as tp  # noqa: E402


def main():
    if not ref_loader.available():
        raise SystemExit("the reference is not importable here")
    ref = ref_loader.load()
    os.makedirs(tp.GOLDEN_DIR, exist_ok=True)
    for name, case in sorted(tp.CASES.items()):
        t = tp.make_inputs(case)
        arrays = {'case': np.array(json.dumps(case, sort_keys=True))}
        arrays.update({'in_' + k: v.numpy() for k, v in t.items() if v is not None})
        adv, value, ret, stats = tp.run_oracle(ref, case, t)
        arrays.update(out_adv=adv.numpy(), out_value=value.numpy(), out_return=ret.numpy())
        if stats is not None:
            arrays['out_stats'] = np.array(stats, np.float64)
        np.savez_compressed(os.path.join(tp.GOLDEN_DIR, name + '.npz'), **arrays)
    print("wrote %d cases to %s" % (len(tp.CASES), tp.GOLDEN_DIR))


if __name__ == '__main__':
    main()
