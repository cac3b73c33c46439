"""Timeline of the column-tile kernel (csrc/colws.cu) at config D: per-CTA %globaltimer stamps of the whole step.

Runs the one-launch step (kernel, finalize_sums, backward check) on rotated buffer sets replayed as one CUDA graph, as
bench.py does, then reads the stamps of the last replay and prints, as median / max over CTAs (us):
  fill    kernel start (earliest CTA) -> the CTA's first chunk landed
  chunk   time per chunk in the middle: (last landed - first landed) / (chunks - 1)
  tail    last chunk landed -> CTA end (partial sums stored)
and the step boundary: one set's kernel end (latest CTA) -> the next set's kernel start and its griddepcontrol.wait
(finalize_sums and the check launch sit between them).  Per SM (median over the SMs that run a CTA of both steps), the
next step's CTA start, wait returned and first chunk landed relative to the end of the previous step's CTA on that SM,
and the share of SMs on which the next step's CTA started before the previous one ended.  --json prints one JSON line
instead of the table.
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
sets = [bench.DeviceStep(bench.make_batch(i), 'cuda:0', fused='onepass') for i in range(NSETS)]
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
tr = trs[0].astype(np.float64)
grid = tr.shape[0]
t0 = tr[:, 0].min()
us = lambda a: (a - t0) / 1e3  # noqa: E731
nch = (trs[0][:, 7] & 0xffffffff).astype(np.int64)
first_landed = us(tr[:, 8])
last_landed = us(tr[:, 3])
end = us(tr[:, 6])
res = {
    'grid': grid,
    'chunks_per_cta': stat(nch),
    'start': stat(us(tr[:, 0])),
    'wait_done': stat(us(tr[:, 1])),
    'fill': stat(first_landed),
    'first_adv_published': stat(us(tr[:, 2])),
    'chunk': stat(np.where(nch > 1, (last_landed - first_landed) / np.maximum(nch - 1, 1), np.nan)),
    'tail': stat(end - last_landed),
    'last_compute': stat(us(tr[:, 5]) - last_landed),
    'kernel_span': round(float(end.max()), 3),
}
# per chunk j (as stamped): landed, advantages ready, computed, issued by the loader
per = {}
for j in range(13):
    c = tr[:, 8 + 4 * j]
    if (c > 0).sum() == 0:
        break
    per[j] = {k: round(float(np.median(us(tr[:, 8 + 4 * j + o][tr[:, 8 + 4 * j + o] > 0]))), 3)
              for o, k in enumerate(('landed', 'adv', 'computed', 'issued'))}
res['per_chunk_median'] = per
# step boundary: kernel end of step k (latest CTA) -> the first CTA of step k+1 starting (PDL launches it early, so this is
# negative) and -> its griddepcontrol.wait returning: finalize_sums and the check launch run in between
res['boundary_end_to_next_start'] = [round(float((b[:, 0].min() - a[:, 6].max()) / 1e3), 3) for a, b in zip(trs[:-1], trs[1:])]
res['boundary_end_to_next_wait_done'] = [round(float((b[:, 1].min() - a[:, 6].max()) / 1e3), 3)
                                         for a, b in zip(trs[:-1], trs[1:])]
res['step_wait_done_to_wait_done'] = [round(float((b[:, 1].min() - a[:, 1].min()) / 1e3), 3)
                                      for a, b in zip(trs[:-1], trs[1:])]


def per_sm(a, b):
    """step a -> step b on each SM that ran a CTA of both: b's start / wait returned / first landed minus a's CTA end (us)"""
    end = {int(r[7]) >> 32: r[6] for r in a}
    rows = [(r[0] - end[s], r[1] - end[s], r[8] - end[s]) for r in b if (s := int(r[7]) >> 32) in end]
    d = np.asarray(rows, dtype=np.float64) / 1e3
    return {'sms': len(rows), 'start': round(float(np.median(d[:, 0])), 3), 'wait_done': round(float(np.median(d[:, 1])), 3),
            'first_landed': round(float(np.median(d[:, 2])), 3),
            'started_before_end': round(float((d[:, 0] < 0).mean()), 3)}


res['per_sm_next_vs_prev_end'] = [per_sm(a, b) for a, b in zip(trs[:-1], trs[1:])]
# the next step's first chunk as its loader saw it land, against its own griddepcontrol.wait returning (negative: it
# landed before the previous step's finalize and check launches had completed)
res['next_first_landed_minus_wait_done'] = [round(float(np.median((b[:, 60] - b[:, 1]) / 1e3)), 3) for b in trs[1:]]
if '--json' in sys.argv:
    print(json.dumps(res))
else:
    for k, v in res.items():
        print('%-32s %s' % (k, v))
