"""Mint the fixtures of ScatterConnection under tests/golden/scatter/ from the UNMODIFIED reference
(oracle/ref_scatter.py), run on the CPU, where its 'cover' is deterministic.

    python tests/golden/make_scatter_golden.py

One ``<case>.npz`` per entry of ``tests.test_scatter_connection.GOLDEN_CASES``: the case parameters (``case``, JSON), the
sums of its seeded inputs (``in_sums``) and upstream gradient (``g_sum``) -- the tests regenerate them from the seeds and
check them against these -- and, for 'add' and 'cover', the map (``<type>_out``) and d x (``<type>_grad_x``) for that
upstream gradient.  A tensor of more than ``SAMPLE`` entries is kept as a seeded sample of them plus its float64 sum
(``<type>_<name>_sum``).
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import ref_scatter  # noqa: E402
from tests import test_scatter_connection as ts  # noqa: E402


def main():
    ref_scatter.build()
    os.makedirs(ts.GOLDEN_DIR, exist_ok=True)
    with ts.reference_cls() as Ref:
        for name in ts.GOLDEN_CASES:
            c = ts.golden_case(name)
            x, index = ts.make_inputs(c)
            g = ts.upstream(c)
            arrays = {'case': np.array(json.dumps(c, sort_keys=True)), 'in_sums': ts.input_sums(x, index),
                      'g_sum': g.double().sum().numpy()}
            for scatter_type in ('add', 'cover'):
                for k, v in zip(('out', 'grad_x'), ts.run(Ref(scatter_type), c, x, index, g, 'cpu')):
                    s, total = ts.sample(v)
                    arrays['%s_%s' % (scatter_type, k)] = s
                    if total is not None:
                        arrays['%s_%s_sum' % (scatter_type, k)] = total
            np.savez_compressed(os.path.join(ts.GOLDEN_DIR, name + '.npz'), **arrays)
    print("wrote %d cases to %s" % (len(ts.GOLDEN_CASES), ts.GOLDEN_DIR))


if __name__ == '__main__':
    main()
