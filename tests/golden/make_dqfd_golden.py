"""Mint the DQfD fixtures under tests/golden/dqfd/ from the UNMODIFIED reference (oracle/ref_loader.py).

    python tests/golden/make_dqfd_golden.py

One ``<case>.npz`` per entry of ``tests.test_dqfd.CASES``: the seeded inputs (``in_*``), the case parameters (``case``, JSON),
the five outputs of ``dqfd_nstep_td_error[_with_rescale]`` (``out_loss``, ``out_per``, ``out_s_n``, ``out_s_1``,
``out_s_je``) and the gradient of q for the upstream mix ``tests.test_dqfd.GRAD_MIX`` on all five (``out_grad_q``).  Also
``ported_test_dqfd_nstep_td.npz``: the values of the reference's own test (ding/rl_utils/tests/test_td.py:403-428) as
ported in tests/test_dqfd.py.  The files live in a subdirectory so that the flat fixture set of tests/golden/*.npz, which
tests/test_oracle.py checks against tests/cases.py, is unchanged.
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import ref_loader  # noqa: E402
from tests import test_dqfd as td  # noqa: E402


def main():
    if not ref_loader.available():
        raise SystemExit("the reference is not importable here")
    ref = ref_loader.load()
    os.makedirs(td.GOLDEN_DIR, exist_ok=True)
    for name, case in sorted(td.CASES.items()):
        t = td.make_inputs(case['seed'], case['B'], case['N'], case['nstep'], case['cum'], case['done'], case['weight'],
                           case['expert'], case['ties'])
        out = td.run(ref, case, t, 'cpu')
        arrays = {'case': np.array(json.dumps(case, sort_keys=True))}
        arrays.update({'in_' + k: v.numpy() for k, v in t.items() if v is not None})
        arrays.update({'out_' + k: v for k, v in out.items()})
        np.savez_compressed(os.path.join(td.GOLDEN_DIR, name + '.npz'), **arrays)
    np.savez_compressed(td.PORT_FILE, **td.ported_body(ref, 'cpu'))
    print("wrote %d cases and the ported test to %s" % (len(td.CASES), td.GOLDEN_DIR))


if __name__ == '__main__':
    main()
