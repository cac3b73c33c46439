"""Timeline of the PPO tile kernel (csrc/ppo.cu) at config P: per-CTA %globaltimer stamps of the learner step.

Runs config P's three calls (gae_returns, ppo forward-with-gradient + finalize_sums, backward check) on rotated buffer sets
replayed as one CUDA graph, as bench.py does, then reads the PPO kernel's stamps of the last replay and prints, as
median / max over CTAs (us):
  fill    the CTA's griddepcontrol.wait returned (the advantage recompute's results visible) -> its first stage landed
  stage   time per stage in the middle: (last landed - first landed) / (stages - 1)
  tail    last stage landed -> CTA end (partial sums stored)
and the boundary: the earliest CTA's wait returned (returns_kernel has completed) -> the first stage landed, and the kernel
span from the earliest wait to the latest end.  --json prints one JSON line instead of the table.
"""
import json
import os
import sys

os.environ['B200RL_FUSED_TRACE'] = '1'
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402

NSETS = 4
wl = bench.WorkloadP()
sets = [wl.device_step(wl.make_batch(i), 'cuda:0') for i in range(NSETS)]
for s in sets[1:]:  # a workspace per set, so that every step of a replay keeps its own stamps
    s.ws = torch.zeros_like(sets[0].ws)
main = torch.cuda.Stream()
with torch.cuda.stream(main):
    for s in sets:
        s()
    main.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=main):
        for s in sets:
            s()
    for _ in range(20):
        g.replay()
    main.synchronize()


def stamps(s):
    ws = s.ws.view(torch.int64)
    tr = ws[65536 // 2: 65536 // 2 + 64 * 512].cpu().numpy().reshape(-1, 64)
    grid = int((tr[:, 0] != 0).sum())
    return tr[:grid]


def stat(x):
    x = np.asarray(x, dtype=np.float64)
    x = x[~np.isnan(x)]
    return {'median': round(float(np.median(x)), 3), 'max': round(float(x.max()), 3), 'min': round(float(x.min()), 3)}


trs = [stamps(s) for s in sets]
res = {'grid': [int(t.shape[0]) for t in trs]}
for key in ('fill', 'stage', 'tail', 'boundary_wait_to_first_landed', 'kernel_span', 'start_to_wait'):
    res[key] = []
for t in trs:
    tr = t.astype(np.float64)
    nst = (t[:, 5] & 0xffffffff).astype(np.int64)
    wait, first, last, end = tr[:, 1], tr[:, 2], tr[:, 3], tr[:, 4]
    res['fill'].append(stat((first - wait) / 1e3))
    res['stage'].append(stat(np.where(nst > 1, (last - first) / np.maximum(nst - 1, 1) / 1e3, np.nan)))
    res['tail'].append(stat((end - last) / 1e3))
    res['boundary_wait_to_first_landed'].append(stat((first - wait.min()) / 1e3))
    res['kernel_span'].append(round(float((end.max() - wait.min()) / 1e3), 3))
    res['start_to_wait'].append(stat((wait - tr[:, 0]) / 1e3))
res['stages_per_cta'] = stat((trs[0][:, 5] & 0xffffffff).astype(np.int64))
# per stage j (median over CTAs, us after the earliest wait of the step)
tr = trs[0].astype(np.float64)
w0 = tr[:, 1].min()
res['landed_median'] = [round(float(np.median((tr[:, 8 + j][tr[:, 8 + j] > 0] - w0) / 1e3)), 3)
                        for j in range(56) if (tr[:, 8 + j] > 0).any()]
if '--json' in sys.argv:
    print(json.dumps(res))
else:
    for k, v in res.items():
        print('%-32s %s' % (k, v))
