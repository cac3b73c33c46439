"""Mint the fixtures of the entropy-regularised TD losses under tests/golden/soft_td/ from the UNMODIFIED reference
(oracle/ref_loader.py).

    python tests/golden/make_soft_td_golden.py

One ``<case>.npz`` per entry of ``tests.test_soft_td.CASES``: the seeded inputs (``in_*``), the case parameters (``case``,
JSON), the outputs of ``m_q_1step_td_error`` / ``q_nstep_sql_td_error`` / ``q_v_1step_td_error`` (``out_*``) and the
gradient of q for the upstream mix of ``tests.test_soft_td.run`` (``out_grad_q``), all computed on the CPU.  Also
``ported_reference_tests.npz``: the values of the reference's own tests (ding/rl_utils/tests/test_td.py:432, :592) as ported
in tests/test_soft_td.py.
"""
import json
import os
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import ref_loader  # noqa: E402
from tests import test_soft_td as st  # noqa: E402


def main():
    if not ref_loader.available():
        raise SystemExit("the reference is not importable here")
    ref = ref_loader.load()
    os.makedirs(st.GOLDEN_DIR, exist_ok=True)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)  # the reference's broadcasting MSELoss and implicit softmax dim
        for name, case in sorted(st.CASES.items()):
            t = st.make_inputs(case)
            out = st.run(ref, case, t, 'cpu')
            arrays = {'case': np.array(json.dumps(case, sort_keys=True))}
            arrays.update({'in_' + k: v.numpy() for k, v in t.items() if v is not None})
            arrays.update({'out_' + k: v for k, v in out.items()})
            np.savez_compressed(os.path.join(st.GOLDEN_DIR, name + '.npz'), **arrays)
        np.savez_compressed(st.PORT_FILE, **st.ported_body(ref, 'cpu'))
    print("wrote %d cases and the ported tests to %s" % (len(st.CASES), st.GOLDEN_DIR))


if __name__ == '__main__':
    main()
