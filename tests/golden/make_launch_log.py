"""Write tests/golden/launch_log.json: the C-ABI launch log of every case of tests/test_launch_log.py, recorded on the CPU
against the logging stand-in for the CUDA library (no GPU needed).

    python tests/golden/make_launch_log.py

One entry per line, so that a change in the launch sequence reads as a short diff.
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests import test_launch_log as tl  # noqa: E402


def main():
    names = sorted(tl.CASES)
    with open(tl.GOLDEN, 'w') as f:
        f.write('{\n')
        for i, name in enumerate(names):
            entries = ',\n'.join('  ' + json.dumps(e) for e in tl.record(name))
            f.write('%s: [\n%s\n]%s\n' % (json.dumps(name), entries, ',' if i + 1 < len(names) else ''))
        f.write('}\n')
    print("wrote %d cases to %s" % (len(names), tl.GOLDEN))


if __name__ == '__main__':
    main()
