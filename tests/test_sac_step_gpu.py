"""
One gradient step of the fused SAC trainer (rl_baselines.sac.train on the GPU), rebuilt in float64 from the ring and the arena the run leaves.

With the defaults (learning_starts 100, batch_size 64) and num_timesteps = 100 N, the run acts uniformly at random for all of its 100 lockstep
steps and takes its only gradient step at the last one, t = 99, eagerly.  train.last_before_first_step holds the arena, the target and the
Adam state before that step, and the ring's first 100 rows are the ring the step sampled from.  So tests/sac_numpy_ref.py can redo the step:
the indices and the reparameterisation noise from the trainer's Philox record (seed + 1 for rank 0, counter 0), the backups, log-probabilities
and every gradient group, and then the Adam step and the Polyak update, which are checked bit for bit from the kernel's own gradient.  That
checks the chain srl_sac_store -> srl_sac_prepare -> srl_sac_grad -> srl_sac_adam as the trainer wires it (the ring arrays each kernel reads,
gamma, the entropy target, the gradient of log_ent_coef written into the arena's last entry, the learning rate, tau), not each kernel alone;
and the ring the 100 collection steps wrote (srl_sac_act's random mode, the filter, srl_sac_store).

Cases: KukaButton at 4096 envs, KukaButton with a stack of 4 (width 12), MobileRobot at 8192 envs; each over the default 50 000-row ring.
"""
import numpy as np
import pytest
import torch

from sac_numpy_ref import sac_step_model
from test_consumer_reference_cpu import grad_bound, philox_words, u53
from test_sac_gpu import _gauss, _tensors

pytestmark = pytest.mark.gpu

T, SEED = 100, 5
RUNS = [("KukaButtonGymEnv-v0", 4096, 1, {}), ("KukaButtonGymEnv-v0", 4096, 4, {}), ("MobileRobotGymEnv-v0", 8192, 1, dict(shape_reward=True))]
IDS = ["%s_%d_stack%d" % (r[0].split("GymEnv")[0], r[1], r[2]) for r in RUNS]
f32 = np.float32


@pytest.fixture(scope="module", params=RUNS, ids=IDS)
def run(request, cuda_lib):
    env_id, N, K, kw = request.param
    from srl_sim import backend
    backend.use_library(None, None)
    from rl_baselines.sac import train
    train(env_id, N, T * N, seed=SEED, env_kwargs=dict(is_discrete=False, **kw), verbose=0, num_stack=K)
    assert train.stats["grad_steps"] == 1 and train.stats["graph_replays"] == 0, train.stats
    nets, (m, v, beta_power) = train.last_nets, train.last_adam
    before = {k: x.cpu().numpy() for k, x in train.last_before_first_step.items()}
    out = dict(N=N, W=nets.obs_dim, A=nets.act_dim, before=before, ring={k: x[:T].cpu().numpy() for k, x in train.last_ring.items()},
               grad=train.last_grad.cpu().numpy(), arena=nets.arena.detach().cpu().numpy(), target=nets.target.cpu().numpy(),
               m=m.cpu().numpy(), v=v.cpu().numpy(), beta_power=beta_power.cpu().numpy(), step=int(train.last_fused["store"].step[0]))
    train.last_ring = train.last_nets = train.last_fused = None      # the 50 000-row ring: free it before the next case
    torch.cuda.empty_cache()
    return out


def _model(r, idx, eps, chunk=1 << 16):
    """sac_step_model over the batch in chunks (each chunk's means rescaled to the whole batch): the float64 gradient arena and q_backup /
    v_backup / logp."""
    from rl_baselines.sac import SAC_DEFAULTS
    W, A, B = r["W"], r["A"], len(idx)
    flat = {k: a.reshape((-1,) + a.shape[2:]) for k, a in r["ring"].items()}
    grad, vals = 0.0, {k: [] for k in ("q_backup", "v_backup", "logp")}
    for lo in range(0, B, chunk):
        ix = idx[lo:lo + chunk]
        g, ref = sac_step_model(r["before"]["arena"], r["before"]["target"], W, A, flat["obs"][ix], flat["act"][ix], flat["rew"][ix], flat["next_obs"][ix],
                                flat["done"][ix].astype(np.float64), eps[lo:lo + chunk], SAC_DEFAULTS["gamma"], None, -float(A))
        grad = grad + g * (len(ix) / B)
        for k in vals:
            vals[k].append(ref[k])
    return grad, {k: np.concatenate(x) for k, x in vals.items()}


def _float32_autograd(r, idx, eps):
    """The torch statement (sac_losses) in float32 on the same samples: float32's own error on them."""
    from rl_baselines.sac import SAC_DEFAULTS, SACNets, sac_losses
    W, A = r["W"], r["A"]
    nets = SACNets(W, A)
    with torch.no_grad():
        nets.arena.copy_(torch.from_numpy(r["before"]["arena"]))
        nets.target.copy_(torch.from_numpy(r["before"]["target"]))
    flat = {k: torch.from_numpy(a.reshape((-1,) + a.shape[2:])) for k, a in r["ring"].items()}
    ix = torch.from_numpy(idx)
    L = sac_losses(nets, flat["obs"][ix], flat["act"][ix], flat["rew"][ix], flat["next_obs"][ix], flat["done"][ix].float(),
                   torch.from_numpy(eps).float(), SAC_DEFAULTS["gamma"], None, -float(A))
    return torch.autograd.grad(L["total"], nets.arena)[0].double().numpy()


def test_ring_holds_the_random_collection(run):
    """obs[t + 1] is next_obs[t] byte for byte (srl_sac_store's obs <- new_obs), and every stored action is srl_sac_act's uniform draw of step t:
    2 (word >> 8) / 2^24 - 1 of the stream (seed, env, t), purpose 28 + k / 4."""
    ring, N, A = run["ring"], run["N"], run["A"]
    assert run["step"] == T
    assert np.array_equal(ring["obs"][1:].view(np.uint32), ring["next_obs"][:-1].view(np.uint32))
    for t in (0, 1, T // 2, T - 1):
        want = np.zeros((N, A))
        for k in range(A):
            w = philox_words(SEED, np.arange(N), t, 28 + k // 4)[:, k % 4].astype(np.float64)
            want[:, k] = 2 * (np.floor(w / 256.0) / 16777216.0) - 1
        assert np.array_equal(ring["act"][t].astype(np.float64), want), t
    assert ring["done"][T - 1].dtype == np.uint8 and np.isfinite(ring["rew"]).all()


def test_gradient_step_matches_float64(run):
    from rl_baselines.sac import ADAM_BETA1, ADAM_BETA2, ADAM_EPS, SAC_DEFAULTS
    N, W, A = run["N"], run["W"], run["A"]
    B, size = SAC_DEFAULTS["batch_size"] * N, T * N
    idx = np.minimum(np.floor(u53(philox_words(SEED + 1, np.arange(B), 0, 30)) * size), size - 1).astype(np.int64)
    eps = _gauss(SEED + 1, np.arange(B), 0, 31, A)
    want, _ = _model(run, idx, eps)
    g32 = _float32_autograd(run, idx, eps)
    g = run["grad"].astype(np.float64)
    print("\nB=%d  max|g - g64| / max|g64|  kernel | float32 autograd:" % B)
    for name, lo, hi in _tensors(W, A):
        scale = np.abs(want[lo:hi]).max()
        err, err32 = np.abs(g[lo:hi] - want[lo:hi]).max(), np.abs(g32[lo:hi] - want[lo:hi]).max()
        print("  %s[%d] %.1e|%.1e" % (name, lo, err / scale, err32 / scale), end="")
        assert scale > 0 and err <= grad_bound(scale) + 4.0 * err32, (name, lo, err, err32, scale)
    print()
    assert abs(g[-1] - want[-1]) <= 1e-5 * (1.0 + abs(want[-1])) + 4.0 * abs(g32[-1] - want[-1])    # d ent_coef_loss / d log_ent_coef
    # one TF Adam step from zero slots and the Polyak update, bit for bit from the kernel's gradient (float32, the kernel's order of roundings)
    gk, p0, t0 = run["grad"], run["before"]["arena"], run["before"]["target"]
    b1, b2, lr, tau = f32(ADAM_BETA1), f32(ADAM_BETA2), f32(SAC_DEFAULTS["learning_rate"]), f32(SAC_DEFAULTS["tau"])
    r1, r2 = f32(1) - b1, f32(1) - b2
    m = (gk - f32(0)) * r1
    v = (gk * gk - f32(0)) * r2
    lr_t = (lr * np.sqrt(f32(1) - b2)) / (f32(1) - b1)
    p1 = p0 - (m * lr_t) / (np.sqrt(v) + f32(ADAM_EPS))
    assert np.array_equal(run["m"], m) and np.array_equal(run["v"], v) and np.array_equal(run["arena"], p1)
    from rl_baselines.sac import net_layout
    lay = net_layout(W, A)
    vf = p1[lay["vf"]["w1"][0]:lay["vf"]["end"]]
    assert np.array_equal(run["target"], (f32(1) - tau) * t0 + tau * vf)
    assert np.array_equal(run["beta_power"], np.array([b1 * b1, b2 * b2], np.float32))
    assert np.all(run["before"]["m"] == 0) and run["arena"][-1] != p0[-1]       # log_ent_coef moved by its own gradient
