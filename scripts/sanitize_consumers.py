"""Each A2C and DQN consumer kernel once, for compute-sanitizer (memcheck, racecheck, synccheck, initcheck):
srl_a2c_grad, srl_clip_rmsprop, srl_dqn_act, srl_dqn_target, srl_dqn_grad, srl_clip_adam, srl_replay_add / _sample (prioritized and uniform) /
_update.  Two shapes: a small one (fewer samples than CTAs), and one where every CTA of dqn_target and of the gradient kernels walks several
chunks (sms 64 3 + 17 samples); the narrow (width 3) and the wide (width 12) instantiations.  Replay: a ring of 10 x 1000 transitions
(16384 leaves: a two-pass rebuild).

  compute-sanitizer --tool memcheck python scripts/sanitize_consumers.py
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "robotics-rl-srl_b200"))
import torch
from srl_sim._abi import load_cuda_library
from srl_sim.policy import FusedA2CGrad, FusedClipAdam, FusedClipRMSprop, FusedDQNAct, FusedDQNGrad, FusedDQNTarget, FusedReplay
from rl_baselines.deepq import DuelingQ
from rl_baselines.ppo2 import MlpPolicy

lib = load_cuda_library()
st = torch.cuda.current_stream().cuda_stream
sms = torch.cuda.get_device_properties(0).multi_processor_count
g = torch.Generator(device="cuda").manual_seed(0)
torch.manual_seed(0)
for width, A in ((3, 6), (12, 6)):
    for B in (33, sms * 64 * 3 + 17):
        rows = B + 7
        obs = torch.randn(rows, width, device="cuda", generator=g)
        act = torch.randint(0, A, (rows,), device="cuda", generator=g)
        idx = torch.randperm(rows, device="cuda", generator=g)[:B].contiguous()
        # A2C: the gradient of an update, then clip_by_global_norm + RMSProp
        pol = MlpPolicy(width, n_actions=A).cuda()
        ret, val = torch.randn(B, device="cuda", generator=g), torch.randn(B, device="cuda", generator=g)
        FusedA2CGrad(lib, pol, B)(None, obs, act, ret, val, 0.01, 0.25, stream=st)
        rms = FusedClipRMSprop(lib, pol, 0.5, 0.99, 1e-5)
        rms.lr.fill_(7e-4)
        rms(stream=st)
        # DQN: act, target, gradient (importance weights and NULL), clip + Adam
        q, qt = DuelingQ(width, A).cuda(), DuelingQ(width, A).cuda()
        fact = FusedDQNAct(lib, q, seed=1)
        fact.eps.fill_(0.3)
        a32, a64, qout, obuf = (torch.zeros(rows, dtype=torch.int32, device="cuda"), torch.zeros(rows, dtype=torch.int64, device="cuda"),
                                torch.zeros(rows, A, device="cuda"), torch.zeros(rows, width, device="cuda"))
        fact(rows, obs, a32, obs_buf=obuf, act_buf=a64, q_out=qout, stream=st)
        rew, done = torch.randn(rows, device="cuda", generator=g), (torch.rand(rows, device="cuda", generator=g) < 0.2).to(torch.uint8)
        y, td, w = torch.zeros(B, device="cuda"), torch.zeros(B, device="cuda"), 0.5 + torch.rand(B, device="cuda", generator=g)
        FusedDQNTarget(lib, q, qt)(B, idx, obs, rew, done, 0.99, y, stream=st)
        fgrad = FusedDQNGrad(lib, q, B)
        fgrad(idx, obs, act, y, w, td, stream=st)
        fgrad(None, obs, act, y, None, td, stream=st)
        adam = FusedClipAdam(lib, q, 10.0)
        adam.lr.fill_(1e-4)
        adam(stream=st)
        torch.cuda.synchronize()
        print("width %d, batch %d: consumer kernels ran" % (width, B))
# replay: adds that wrap the ring, a prioritized and a uniform batch, the priorities
rep = FusedReplay(lib, 10, 1000, 2, 0.6, "cuda")
B = 4096
ix, wt = torch.zeros(B, dtype=torch.int64, device="cuda"), torch.zeros(B, device="cuda")
for step in range(12):
    rep.add(step % 10, stream=st)
    if step >= 2:
        rep.beta.fill_(0.5)
        rep.sample(B, ix, wt, prioritized=bool(step % 2), stream=st)
        rep.update(B, ix, torch.randn(B, device="cuda", generator=g), 1e-6, stream=st)
torch.cuda.synchronize()
print("replay: root %.6g, size %d" % (float(rep.sum[1]), int(rep.size)))
