"""Mint the fixtures of the continuous-action policy-gradient losses under tests/golden/pg_continuous/ from the UNMODIFIED
reference (oracle/ref_loader.py).

    python tests/golden/make_pg_continuous_golden.py

One ``<case>.npz`` per entry of ``tests.test_pg_continuous.CASES``: the seeded inputs (``in_*``), the case parameters
(``case``, JSON), the outputs of ``a2c_error_continuous`` / ``ppo_policy_error_continuous`` (``out_*``) and the gradients of
mu, sigma (and value) for the upstream mix of ``tests.test_pg_continuous.run`` (``out_grad_*``), all computed on the CPU.
Also ``ported_reference_tests.npz``: the values of the reference's own ``test_a2c_continuous``
(ding/rl_utils/tests/test_a2c.py:31-54) as ported in tests/test_pg_continuous.py.
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import ref_loader  # noqa: E402
from tests import test_pg_continuous as pc  # noqa: E402


def main():
    if not ref_loader.available():
        raise SystemExit("the reference is not importable here")
    ref = ref_loader.load()
    os.makedirs(pc.GOLDEN_DIR, exist_ok=True)
    for name, case in sorted(pc.CASES.items()):
        t = pc.make_inputs(case)
        out = pc.run(ref, case, t, 'cpu')
        arrays = {'case': np.array(json.dumps(case, sort_keys=True))}
        arrays.update({'in_' + k: v.numpy() for k, v in t.items() if v is not None})
        arrays.update({'out_' + k: v for k, v in out.items()})
        np.savez_compressed(os.path.join(pc.GOLDEN_DIR, name + '.npz'), **arrays)
    np.savez_compressed(pc.PORT_FILE, **pc.ported_body(ref, 'cpu'))
    print("wrote %d cases and the ported test to %s" % (len(pc.CASES), pc.GOLDEN_DIR))


if __name__ == '__main__':
    main()
