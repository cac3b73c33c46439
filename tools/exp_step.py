"""Time the learner step variants at config D's shape: ppo_fwd_grad, ppo_fwd and gae alone, the one-launch step, and the
three-launch and one-launch steps with their backward check."""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench
from tools.bench_ops import timed
res = {}
sets = [bench.DeviceStep(bench.make_batch(i), 'cuda:0', fused=True) for i in range(6)]
for s in sets:
    s.gae()
torch.cuda.synchronize()
res['ppo_fwd_grad_us'] = round(timed([s.ppo_fwd_grad for s in sets], reps=30), 2)
res['ppo_fwd_us'] = round(timed([s.ppo_fwd for s in sets], reps=30), 2)
res['gae_us'] = round(timed([s.gae for s in sets], reps=30), 2)
res['onepass_us'] = round(timed([s.gae_ppo_fwd_grad for s in sets], reps=30), 2)
def three(s):
    s.gae(); s.ppo_fwd_grad(); s.ppo_bwd_check()
def one(s):
    s.gae_ppo_fwd_grad(); s.ppo_bwd_check()
res['step3_us'] = round(timed([lambda s=s: three(s) for s in sets], reps=30), 2)
res['step1_us'] = round(timed([lambda s=s: one(s) for s in sets], reps=30), 2)
print(json.dumps(res))
