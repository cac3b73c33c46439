"""Mint the fixtures of COMA's loss under tests/golden/coma/ from the UNMODIFIED reference (oracle/ref_coma.py, whose
``generalized_lambda_returns`` is the reference's own, oracle/ref_loader.py).

    python tests/golden/make_coma_golden.py

One ``<case>.npz`` per entry of ``tests.test_coma.CASES``: the case parameters (``case``, JSON), the sums of its seeded
inputs (``in_sums``: the tests regenerate the inputs and check them against these), the three losses and d (policy + value +
entropy loss) / d logit, q_value, target_q_value and reward (``out_*``), computed by ``coma_error``
(ding/rl_utils/coma.py:10-58) on the CPU with every input but action and weight requiring grad.  A gradient of more than
``tests.test_coma.FULL_MAX`` entries is kept as a seeded sample of them plus its float64 sum (``sum_*``).
``ported_reference_test.npz`` holds the reference's losses and gradients in ding/rl_utils/tests/test_coma.py, for weight
None (``none_*``) and its random weight (``random_*``).
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import ref_coma  # noqa: E402
from tests import test_coma as tc  # noqa: E402


def ported(ref):
    """what the reference computes in ding/rl_utils/tests/test_coma.py, for weight None and its random weight"""
    arrays = {}
    for name, inputs in tc.ported_inputs().items():
        arrays.update({name + '_' + k: v for k, v in tc.pack(tc.ported_test(ref.coma_data, ref.coma_error, inputs,
                                                                            'cpu')).items()})
    return arrays


def main():
    ref_coma.build()
    os.makedirs(tc.GOLDEN_DIR, exist_ok=True)
    with ref_coma.module() as ref:
        for name, case in sorted(tc.CASES.items()):
            t = tc.make_inputs(case)
            arrays = {'case': np.array(json.dumps(case, sort_keys=True))}
            arrays['in_sums'] = tc.input_sums(t)
            arrays.update(tc.pack(tc.run(ref.coma_error, ref.coma_data, t, 'cpu', case)))
            np.savez_compressed(os.path.join(tc.GOLDEN_DIR, name + '.npz'), **arrays)
        np.savez_compressed(os.path.join(tc.GOLDEN_DIR, 'ported_reference_test.npz'), **ported(ref))
    print("wrote %d cases to %s" % (len(tc.CASES) + 1, tc.GOLDEN_DIR))


if __name__ == '__main__':
    main()
