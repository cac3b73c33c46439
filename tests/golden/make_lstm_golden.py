"""Mint the fixtures of the layer-normalised LSTM under tests/golden/lstm/ from the UNMODIFIED reference
(ding/torch_utils/network/rnn.py, through oracle/ref_scatter.py's archive), run in fp32 on the CPU.

    python tests/golden/make_lstm_golden.py

One ``<case>.npz`` per entry of ``tests.test_lstm.GOLDEN_CASES``: the case parameters (``case``, JSON), the sums of its
seeded inputs and upstream gradients (``in_sums``) and of the seeded initial weights (``w_sums``) -- the tests regenerate
them from the seeds and check them against these -- and the reference's output, next state and every gradient
(``ref_<name>``, as ``tests.test_lstm.run`` names them).
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import ref_scatter  # noqa: E402
from tests import test_lstm as tl  # noqa: E402


def main():
    ref_scatter.build()
    os.makedirs(tl.GOLDEN_DIR, exist_ok=True)
    with tl.reference_rnn() as rnn:
        for name in tl.GOLDEN_CASES:
            c = tl.GOLDEN[name]
            ref = tl.ref_model(rnn, c)
            arrays = {'case': np.array(json.dumps(c, sort_keys=True)), 'in_sums': tl.input_sums(c),
                      'w_sums': np.array([float(v.double().sum()) for v in ref.state_dict().values()])}
            for k, v in tl.run(ref, c, 'cpu').items():
                arrays['ref_' + k] = v.astype(np.float32)
            np.savez_compressed(os.path.join(tl.GOLDEN_DIR, name + '.npz'), **arrays)
    print("wrote %d cases to %s" % (len(tl.GOLDEN_CASES), tl.GOLDEN_DIR))


if __name__ == '__main__':
    main()
