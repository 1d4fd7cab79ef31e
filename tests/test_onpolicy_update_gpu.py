"""
One update of the fused PPO2 and A2C trainers (rl_baselines.ppo2.train, rl_baselines.a2c.train on the GPU, fused paths and CUDA graphs on),
rebuilt in float64 from what the run leaves behind (``train.last_update``).  The kernels are each held to float64 in their own tests; this
file checks how the trainers wire them together:
  the simulator   -- the envs rebuilt with the same seed and kwargs and stepped eagerly with the trainer's actions give its rewards, dones and
                     episode statistics byte for byte, and the raw observations the filter saw;
  the filter      -- obs[t] is the float64 filter chain (the reset batch, then one merge per step; with a stack, the stack of raw frames zeroed
                     where done), and the final filter state is the chain's;
  the draws       -- every action is sample_model's at counter t (A2C's second half: T + t), under the float64 policy at the buffer's own obs[t];
                     logp[t], val[t] and last_val match the float64 towers;
  GAE             -- adv / ret are gae_model on the buffers, lambda 0.95 (PPO2) and 1 (A2C);
  the optimiser   -- PPO2: the clipped gradient, Adam's moments and the parameter move of one step over all rows; the moments after 16 minibatch
                     steps whose indices come from the run's permutations.  A2C: two updates of one graph replay at the two learning rates of a
                     linear schedule, against a2c_grads_model + clip_rmsprop_model; and one eager update.
Finally a captured and an eager PPO2 run of two updates agree to float32 rounding.
"""
import copy
import types

import numpy as np
import pytest
import torch

from a2c_numpy_ref import a2c_grads_model, clip_rmsprop_model, scheduler_values
from test_consumer_kernels_gpu import check_draws
from test_consumer_reference_cpu import (GAE_ULPS, clip_adam_torch_model, clip_grad_norm_model, filter_model, gae_model, grad_bound, grad_errors,
                                         logp_model, normalise, policy_model, ppo2_minibatch_grads)

pytestmark = pytest.mark.gpu

N, SEED = 4096, 3
MAX_NORM = 0.5
# Episodes of 7 steps end inside every rollout (steps 6 and 13 of PPO2's 16, steps 2 and 4 of A2C's two halves of 5 at max_steps 3): GAE's
# masking, the bootstrap at a done last step and the stack's zeroing all run.
MOBILE = ("MobileRobotGymEnv-v0", dict(is_discrete=True, shape_reward=True, max_steps=7))
KUKA_D = ("KukaButtonGymEnv-v0", dict(is_discrete=True, max_steps=7))
KUKA_B = ("KukaButtonGymEnv-v0", dict(is_discrete=False, max_steps=7))
KUKA_J = ("KukaButtonGymEnv-v0", dict(is_discrete=False, action_joints=True, max_steps=7))


def _np(t):
    return t.detach().cpu().numpy()


def _with_params(template, params, dtype=torch.float32):
    """A copy of the trainer's policy holding ``params`` (tensors or arrays in parameters() order), in ``dtype``."""
    pol = copy.deepcopy(template).to(dtype)
    with torch.no_grad():
        for p, v in zip(pol.parameters(), params):
            p.copy_(torch.as_tensor(np.asarray(v) if not torch.is_tensor(v) else v, dtype=dtype))
            p.grad = None                    # the trainer's static .grad tensors came with the copy: autograd must not add to them
    return pol


# ---------------------------------------------------------------- the collection, shared by both trainers

def _replay(env_id, env_kwargs, K, acts):
    """The trainer's envs rebuilt (createTensorEnvs with the same seed and kwargs, next-episode records on as make_run sets them) and stepped
    eagerly with ``acts``: the raw observations after the reset and after every step, and each step's rew / done / ep_ret / ep_len."""
    from rl_baselines.utils import createTensorEnvs
    env = createTensorEnvs(types.SimpleNamespace(env=env_id, num_cpu=N, seed=SEED, device=0), env_kwargs=dict(env_kwargs, prefetch_resets=True))
    st = env.backend.stream()
    env.sim.reset(obs_out=env._obs, stream=st)             # the order of first_observation, then the trainer's bulk fill of the records
    env.sim.prefetch_resets(stream=st)
    raws, outs = [env._obs.clone()], []
    for a in acts:
        env.sim.step(a.contiguous(), None, env._obs, env._rew, env._done, env._ep_ret, env._ep_len, stream=st)
        raws.append(env._obs.clone())
        outs.append([env._rew.clone(), env._done.clone(), env._ep_ret.clone(), env._ep_len.clone()])
    torch.cuda.synchronize()
    env.close()
    return [_np(r) for r in raws], [[_np(x) for x in o] for o in outs]


def _filter_chain(raws, dones, K):
    """The rows the filter sees (the raw observation, or the frame stack: zeros and the first frame at the reset, then roll, zero where the step
    ended an episode and insert) and the float64 filter state after each merge."""
    D = raws[0].shape[1]
    W = K * D
    state = np.concatenate([np.zeros(W), np.ones(W), [1e-4]])
    stack = np.zeros((N, W), np.float32)
    rows, states = [], []
    for t, x in enumerate(raws):
        if K > 1:
            stack = np.roll(stack, -D, 1) if t else np.zeros_like(stack)
            if t:
                stack[dones[t - 1].astype(bool)] = 0.0
            stack[:, W - D:] = x
            row = stack.copy()
        else:
            row = x
        state = filter_model(state, row)
        rows.append(row)
        states.append(state)
    return rows, states


def _normalise_bound(row, state, want):
    """A float32 output of the filter on a state within the filter tests' tolerance (1e-11) of the model's: the float32 mean may round one
    ulp apart and move by 1e-11 (moving the output by that over std), the variance by 1e-11 (moving it by |out| 1e-11 / (2 (var + eps)): a column
    that barely varies, such as the zeroed frames of a stack, amplifies it), and the division and the square root add a few ulps."""
    W = row.shape[1]
    var = state[W:2 * W] + 1e-8
    std = np.sqrt(var.astype(np.float32))
    return ((2.0 * np.spacing(np.abs(state[:W]).astype(np.float32)) + 1e-11) / std + np.abs(want) * 0.5e-11 / var
            + 4.0 * np.spacing(np.abs(want)))


def check_collection(env_id, env_kwargs, K, seed, buf, obs_final, state_final, pols, counter0, last_val, extra_tol=0.0):
    """Every check of a rollout of H halves (``buf`` [H, T, N, ...] numpy; ``pols[h]``: the float64 policy half h ran under; half h drew at
    counters counter0[h] + t).  Returns the share of dones."""
    H, T = buf["rew"].shape[:2]
    discrete = buf["act"].dtype == np.int64
    acts = []
    for h in range(H):
        for t in range(T):
            a = buf["act"][h, t]
            acts.append(torch.from_numpy(a.astype(np.int32) if discrete else np.clip(a, -1.0, 1.0)).cuda())
    raws, outs = _replay(env_id, env_kwargs, K, acts)
    for i, (rew, done, ep_ret, ep_len) in enumerate(outs):
        h, t = divmod(i, T)
        d = done.astype(bool)                                  # the episode statistics are written where an episode ended
        for name, got, want in (("rew", buf["rew"][h, t], rew), ("done", buf["done"][h, t], done.astype(np.float32)),
                                ("ep_ret", buf["ep_ret"][h, t][d], ep_ret[d]), ("ep_len", buf["ep_len"][h, t][d], ep_len[d])):
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (name, h, t, int((got != want).sum()))
    dones = [o[1] for o in outs]
    rows, states = _filter_chain(raws, dones, K)
    W = rows[0].shape[1]
    for i in range(H * T + 1):
        want = _np(normalise(torch.from_numpy(rows[i]), torch.from_numpy(states[i])))
        got = buf["obs"][divmod(i, T)] if i < H * T else obs_final
        err = np.abs(got - want)
        assert (err <= _normalise_bound(rows[i], states[i], want)).all(), (i, err.max())
    s = _np(state_final)
    assert np.allclose(s[:W], states[-1][:W], rtol=0, atol=1e-11) and np.allclose(s[W:2 * W], states[-1][W:2 * W], rtol=1e-11, atol=1e-11)
    assert s[2 * W] == pytest.approx(states[-1][2 * W], rel=1e-14)

    near = 0
    for h in range(H):
        pol = pols[h]
        sigma = None if discrete else np.exp(_np(pol.logstd).astype(np.float64))
        for t in range(T):
            obs_t = buf["obs"][h, t]
            out64, v64 = policy_model(pol, obs_t)
            act = buf["act"][h, t]
            near += check_draws(out64, sigma, seed, np.arange(N), counter0[h] + t, np.clip(act, -1.0, 1.0), act, label="h%d t%d: " % (h, t))
            lp, lp64 = buf["logp"][h, t], logp_model(pol, out64, act)
            if discrete:
                tol = 4e-6 + 1e-6 * np.abs(out64).max(1)
            else:     # the tolerance of test_policy_act_against_a_float64_model
                z = (act.astype(np.float64) - out64) / sigma
                tol = 4e-6 + 4e-7 * (np.abs(z) * (1.0 + np.abs(act)) / sigma).sum(1)
            tol = tol * (1.0 + extra_tol) + extra_tol * 1e-5 * (1.0 + np.abs(out64).max(1))
            assert (np.abs(lp - lp64) <= tol).all(), (h, t, np.abs(lp - lp64).max())
            vtol = (2e-5 + 1e-6 * np.abs(v64)) * (1.0 + extra_tol) + extra_tol * 1e-5 * (1.0 + np.abs(v64))
            assert (np.abs(buf["val"][h, t] - v64) <= vtol).all(), (h, t, np.abs(buf["val"][h, t] - v64).max())
        nxt = buf["obs"][h + 1, 0] if h + 1 < H else obs_final
        _, lv64 = policy_model(pol, nxt)
        vtol = (2e-5 + 1e-6 * np.abs(lv64)) * (1.0 + extra_tol) + extra_tol * 1e-5 * (1.0 + np.abs(lv64))
        assert (np.abs(last_val[h] - lv64) <= vtol).all(), (h, np.abs(last_val[h] - lv64).max())
    share = float(buf["done"].mean())
    print("\n  %d draws within rounding of a CDF boundary; %.1f %% of the steps ended an episode" % (near, 100 * share))
    assert share >= 0.05
    return share


def check_gae(buf, last_val, adv, ret, lam):
    """adv / ret within GAE_ULPS float32 ulps of gae_model.  The ulps are of the recursion's terms (rewards and values, which in a short rollout
    from the initial policy can be larger than the advantages they leave), as well as of the result."""
    for h in range(buf["rew"].shape[0]):
        a64, r64 = gae_model(buf["rew"][h], buf["val"][h], buf["done"][h], last_val[h], 0.99, lam)
        terms = max(np.abs(buf["rew"][h]).max(), np.abs(buf["val"][h]).max(), np.abs(last_val[h]).max())
        for got, want in ((adv[h], a64), (ret[h], r64)):
            assert np.abs(got - want).max() <= GAE_ULPS * 2.0 ** -23 * max(np.abs(want).max(), terms), (h, np.abs(got - want).max())


def _clip_errors(g64, bounds):
    """Per tensor, the bound of |clipped float32 gradient - clipped float64 gradient| elementwise: the clip factor c times the gradient's bound,
    plus |c' - c| |g|, where |c' - c| <= c |g' - g| / |g| and |g' - g| is at most the norm of every entry off by its tensor's bound."""
    gc, c = clip_grad_norm_model(g64, MAX_NORM)
    norm = np.sqrt(sum(float((g ** 2).sum()) for g in g64))
    dg = np.sqrt(sum(b * b * g.size for g, b in zip(g64, bounds)))
    dc = c * dg / max(norm - dg, 1e-30)
    return gc, c, [c * b + dc * np.abs(g) for g, b in zip(g64, bounds)]


# ---------------------------------------------------------------- PPO2

PPO2_CASES = [(MOBILE, 1), (KUKA_B, 1), (KUKA_J, 1), (KUKA_D, 4)]
PPO2_PARAMS = [(c, cfg) for c in PPO2_CASES for cfg in ("one_step", "sixteen_steps")]
PPO2_IDS = ["%s_%s_stack%d-%s" % (c[0][0].split("GymEnv")[0], "discrete" if c[0][1]["is_discrete"] else "box%d" % (7 if c[0][1].get("action_joints") else 3),
                                  c[1], cfg) for c, cfg in PPO2_PARAMS]
T_PPO2 = 16


@pytest.fixture(scope="module", params=PPO2_PARAMS, ids=PPO2_IDS)
def ppo2_run(request, cuda_lib):
    ((env_id, env_kwargs), K), cfg = request.param
    from srl_sim import backend
    backend.use_library(None, None)
    from rl_baselines import ppo2
    hp = dict(n_steps=T_PPO2) if cfg == "sixteen_steps" else dict(n_steps=T_PPO2, nminibatches=1, noptepochs=1)
    if cfg == "sixteen_steps":
        hp["learning_rate"] = 1e-7
    ppo2.train(env_id, N, N * T_PPO2, seed=SEED, env_kwargs=env_kwargs, verbose=0, hyperparams=hp, num_stack=K)
    u = ppo2.train.last_update
    pol = ppo2.train.last_policy
    opt = u["opt"]
    return dict(env_id=env_id, env_kwargs=env_kwargs, K=K, cfg=cfg, lr=ppo2.PPO2_DEFAULTS["learning_rate"] if cfg == "one_step" else 1e-7,
                template=copy.deepcopy(pol), params0=[t.clone() for t in u["params0"]], buf={k: v.clone() for k, v in u["buf"].items()},
                obs=u["obs"].clone(), state=ppo2.train.last_norm.state.clone(), adv=u["adv"].clone(), ret=u["ret"].clone(),
                last_val=u["last_val"].clone(), perms=[p.clone() for p in u["perms"]], mb=u["mb"],
                after=[p.detach().clone() for p in pol.parameters()], grad=[p.grad.detach().clone() for p in pol.parameters()],
                m=[opt.state[p]["exp_avg"].clone() for p in pol.parameters()], v=[opt.state[p]["exp_avg_sq"].clone() for p in pol.parameters()],
                step=[float(opt.state[p]["step"]) for p in pol.parameters()])


def test_ppo2_collection_and_gae(ppo2_run):
    r = ppo2_run
    buf = {k: _np(v)[None] for k, v in r["buf"].items()}
    pol64 = _with_params(r["template"], r["params0"], torch.float64).cpu()
    check_collection(r["env_id"], r["env_kwargs"], r["K"], SEED, buf, _np(r["obs"]), r["state"], [pol64], [0], _np(r["last_val"])[None])
    check_gae(buf, _np(r["last_val"])[None], _np(r["adv"])[None], _np(r["ret"])[None], 0.95)


def _minibatch_grads(r, idx):
    """(float64 gradient, float32 autograd's error per tensor) of one minibatch at the initial parameters."""
    T = T_PPO2
    flat = lambda t: t.reshape((T * N,) + t.shape[2:])
    b = r["buf"]
    d = dict(obs=flat(b["obs"]), act=flat(b["act"]), adv=r["adv"].reshape(-1), ret=r["ret"].reshape(-1), old_logp=flat(b["logp"]), old_val=flat(b["val"]))
    pol32 = _with_params(r["template"], r["params0"]).cuda()
    g64 = ppo2_minibatch_grads(_with_params(r["template"], r["params0"], torch.float64).cuda(), idx, d)
    e32 = grad_errors(ppo2_minibatch_grads(pol32, idx, d), g64)
    return [_np(g) for g in g64], e32


def test_ppo2_optimiser_step(ppo2_run):
    """(one_step) The clipped gradient left in .grad within grad_bound + 4 x float32 autograd's error (through the clip), Adam's first moments and
    the parameter move of about lr sign(g).  (sixteen_steps) Adam's moments after 16 minibatch steps at lr 1e-7 against the float64 weighted sums
    of the 16 clipped minibatch gradients at the initial parameters (the parameters move by at most ~16 lr: their effect on the gradients is far
    below the bound), each minibatch read from the run's permutations."""
    r = ppo2_run
    names = [n for n, _ in r["template"].named_parameters()]
    p0 = [_np(p).astype(np.float64) for p in r["params0"]]
    got_m, got_v = [_np(t).astype(np.float64) for t in r["m"]], [_np(t).astype(np.float64) for t in r["v"]]
    b1, b2 = 0.9, 0.999
    if r["cfg"] == "one_step":
        assert r["mb"] == T_PPO2 * N and len(r["perms"]) == 1 and r["step"] == [1.0] * len(p0)
        g64, e32 = _minibatch_grads(r, r["perms"][0])
        bounds = [grad_bound(float(np.abs(g).max())) + 4.0 * e for g, (e, _) in zip(g64, e32)]
        gc, c, errs = _clip_errors(g64, bounds)
        lr = r["lr"]
        move = lambda g: lr * g / (np.abs(g) + 1e-5)           # Adam's first step: m_hat = g, v_hat = g^2
        print("\n  clip factor %.4f;  max|g - g64| / max|g64|  kernel | float32 autograd:" % c)
        kern = grad_errors([r["grad"][k].cpu() for k in range(len(p0))], [torch.from_numpy(g) for g in gc])
        for k, name in enumerate(names):
            grad = _np(r["grad"][k]).astype(np.float64)
            e = errs[k]
            print("  %s %.1e|%.1e" % (name, kern[k][0] / max(kern[k][1], 1e-30), e32[k][0] / max(e32[k][1], 1e-30)), end="")
            assert (np.abs(grad - gc[k]) <= e).all(), (name, np.abs(grad - gc[k]).max(), e.max())
            # the moments are (1 - beta) g and (1 - beta2) g^2 of the kernel's clipped gradient, which lies within e of the model's
            assert (np.abs(got_m[k] / (1 - b1) - gc[k]) <= e + 4e-7 * np.abs(gc[k])).all(), name
            assert (np.abs(got_v[k] / (1 - b2) - gc[k] ** 2) <= e * (2 * np.abs(gc[k]) + e) + 4e-7 * gc[k] ** 2).all(), name
            p1 = _np(r["after"][k]).astype(np.float64)
            got, ulp = p0[k] - p1, np.spacing(np.abs(p0[k]).astype(np.float32)).astype(np.float64)
            clear = np.abs(gc[k]) > e
            spread = np.maximum(np.abs(move(gc[k] + e) - move(gc[k])), np.abs(move(gc[k] - e) - move(gc[k])))
            assert np.all(np.abs(got - move(gc[k]))[clear] <= spread[clear] + ulp[clear] + 1e-5 * lr), name
            assert np.all(np.abs(got) <= lr * (1.0 + 1e-5) + ulp), name
            assert clear.mean() > 0.2, (name, clear.mean())             # a good share of the entries is compared with the model
        print()
        return
    mb = r["mb"]
    assert mb == T_PPO2 * N // 4 and len(r["perms"]) == 4 and r["step"] == [16.0] * len(p0)
    grads, errs = [], []
    for perm in r["perms"]:
        for s in range(0, T_PPO2 * N, mb):
            g64, e32 = _minibatch_grads(r, perm[s:s + mb])
            _, _, e = _clip_errors(g64, [grad_bound(float(np.abs(g).max())) + 4.0 * x for g, (x, _) in zip(g64, e32)])
            grads.append(g64)
            errs.append(e)
    _, m64, v64, gcs = clip_adam_torch_model(p0, grads, r["lr"], MAX_NORM)
    w1 = [(1 - b1) * b1 ** (15 - s) for s in range(16)]
    w2 = [(1 - b2) * b2 ** (15 - s) for s in range(16)]
    apart = 0.0
    for k, name in enumerate(names):
        em = sum(w * e[k] for w, e in zip(w1, errs)) + 4e-7 * sum(w * np.abs(g[k]) for w, g in zip(w1, gcs))
        ev = sum(w * e[k] * (2 * np.abs(g[k]) + e[k]) for w, e, g in zip(w2, errs, gcs)) + 4e-7 * sum(w * g[k] ** 2 for w, g in zip(w2, gcs))
        assert (np.abs(got_m[k] - m64[k]) <= em).all(), (name, np.abs(got_m[k] - m64[k]).max(), em.max())
        assert (np.abs(got_v[k] - v64[k]) <= ev).all(), (name, np.abs(got_v[k] - v64[k]).max(), ev.max())
        apart = max(apart, float((np.abs(w1[15] * (gcs[14][k] - gcs[15][k])) / em).max()))
        moved = np.abs(_np(r["after"][k]).astype(np.float64) - p0[k]).max()
        assert moved <= 16 * 4 * r["lr"] + np.spacing(np.float32(np.abs(p0[k]).max())), (name, moved)
    # the bound tells the minibatches apart: with step 15's gradient in place of step 16's, the first moment leaves it
    print("\n  another minibatch in place of the last one: %.1f x the bound on the first moment" % apart)
    assert apart > 1.0


def test_ppo2_captured_and_eager_updates_agree(cuda_lib):
    """Two updates captured (collection, GAE and minibatch graphs) and the same two updates launched eagerly draw the same actions and permutations,
    so the actions of the second rollout are the same and the parameters and Adam's moments agree to float32 rounding, carried through 32
    Adam steps.  The captured run steps torch's capturable Adam and the eager one its host-counted Adam, whose float32 roundings differ by an
    ulp; Adam divides by sqrt(v), so an ulp in a small gradient entry moves a parameter by up to ~lr x 1e-7 / |g|, and the second update then
    differentiates at parameters that far apart.  Measured on an H100 (MobileRobot): 2.3e-5 of a tensor's largest entry for the parameters, 6e-5
    for the moments; the bounds are 1e-4 and 5e-4.  A run that draws other actions (the sampling counter) differs in about half of them."""
    from srl_sim import backend
    backend.use_library(None, None)
    from rl_baselines import ppo2
    for (env_id, env_kwargs), K in ((MOBILE, 1), (KUKA_D, 4)):
        out = []
        for graph in (True, False):
            ppo2.train(env_id, N, N * T_PPO2 * 2, seed=SEED, env_kwargs=env_kwargs, verbose=0, hyperparams=dict(n_steps=T_PPO2), num_stack=K,
                       cuda_graph=graph)
            pol, opt = ppo2.train.last_policy, ppo2.train.last_update["opt"]
            out.append([p.detach().clone() for p in pol.parameters()] + [opt.state[p][k].clone() for p in pol.parameters() for k in ("exp_avg", "exp_avg_sq")]
                       + [ppo2.train.last_update["buf"]["act"].clone()])
        equal = all(torch.equal(a, b) for a, b in zip(*out))
        print("\ncaptured vs eager PPO2 (%s, num_stack %d): %s" % (env_id, K, "identical bytes" if equal else "differ"))
        mismatch = float((out[0][-1] != out[1][-1]).float().mean())
        rel = [float((a - b).abs().max()) / float(b.abs().max()) for a, b in zip(out[0][:-1], out[1][:-1])]
        print("  second rollout: %.1e of the actions differ; largest difference / largest entry: parameters %.1e, moments %.1e"
              % (mismatch, max(rel[:len(rel) // 3]), max(rel[len(rel) // 3:])))
        assert mismatch < 1e-3                                      # the second rollouts drew the same actions
        assert max(rel[:len(rel) // 3]) <= 1e-4 and max(rel[len(rel) // 3:]) <= 5e-4


# ---------------------------------------------------------------- A2C

A2C_CASES = [(MOBILE, 1), (KUKA_B, 1), (KUKA_D, 3)]
A2C_PARAMS = [(c, n) for c in A2C_CASES for n in (2, 1)]
A2C_IDS = ["%s_%s_stack%d-%s" % (c[0][0].split("GymEnv")[0], "discrete" if c[0][1]["is_discrete"] else "box", c[1],
                                 "two_updates_one_replay" if n == 2 else "one_eager_update") for c, n in A2C_PARAMS]
T_A2C = 5


@pytest.fixture(scope="module", params=A2C_PARAMS, ids=A2C_IDS)
def a2c_run(request, cuda_lib):
    ((env_id, env_kwargs), K), n_up = request.param
    env_kwargs = dict(env_kwargs, max_steps=3)
    from srl_sim import backend
    backend.use_library(None, None)
    from rl_baselines import a2c
    n_batch = N * T_A2C
    total = 3 * n_batch - 1 if n_up == 2 else 2 * n_batch - 1        # linear schedule: lr x ~2/3 then ~1/3; one update at ~1/2
    hist = a2c.train(env_id, N, total, seed=SEED, env_kwargs=env_kwargs, verbose=0, hyperparams=dict(lr_schedule="linear"), num_stack=K)
    assert len(hist) == n_up
    u, pol = a2c.train.last_update, a2c.train.last_policy
    from srl_sim.policy import policy_params
    slots = dict(zip([id(p) for p in policy_params(pol)], a2c.train.last_ms))     # the slots are in srl_mlp_grads order (logstd last)
    return dict(env_id=env_id, env_kwargs=env_kwargs, K=K, n_up=n_up, total=total, template=copy.deepcopy(pol),
                params0=[t.clone() for t in u["params0"]], buf={k: v[:n_up].clone() for k, v in u["buf"].items()}, obs=u["obs"].clone(),
                state=a2c.train.last_norm.state.clone(), adv=u["adv"][:n_up].clone(), ret=u["ret"][:n_up].clone(), last_val=u["last_val"][:n_up].clone(),
                lr_t=_np(u["lr_t"]).copy(), after=[p.detach().clone() for p in pol.parameters()], grad=[p.grad.detach().clone() for p in pol.parameters()],
                ms=[slots[id(p)].clone() for p in pol.parameters()])


def test_a2c_updates(a2c_run):
    """Half h drew at counters h T + t under the parameters of update h; its returns are GAE with lambda 1; the gradient of the last update
    (left in .grad) within grad_bound + 4 x float32 autograd's error of a2c_grads_model; the final parameters and RMSProp slots within the
    propagated gradient bounds of clip_rmsprop_model applied once per update at the schedule's learning rates."""
    from rl_baselines.a2c import A2C_DEFAULTS, a2c_loss
    r = a2c_run
    hp = A2C_DEFAULTS
    n_up, T = r["n_up"], T_A2C
    lrs = scheduler_values(hp["learning_rate"], r["total"], "linear", N * T, n_up)
    assert np.allclose(r["lr_t"][:n_up], lrs, rtol=1e-6, atol=0) and (n_up == 1 or lrs[0] > 1.5 * lrs[1])
    names = [n for n, _ in r["template"].named_parameters()]
    buf = {k: _np(v) for k, v in r["buf"].items()}
    ret = _np(r["ret"])
    # float64 updates, each from the previous one's float64 parameters
    params, ms = [[_np(p).astype(np.float64) for p in r["params0"]]], [np.ones(p.shape) for p in r["params0"]]
    grads, bounds = [], []
    for h in range(n_up):
        pol64 = _with_params(r["template"], params[h], torch.float64).cuda()
        x = lambda k: buf[k][h].reshape((T * N,) + buf[k].shape[3:])
        g64 = a2c_grads_model(pol64, x("obs"), x("act"), ret[h].reshape(-1), x("val"), hp["ent_coef"], hp["vf_coef"])
        pol32 = _with_params(r["template"], params[h]).cuda()
        act = torch.from_numpy(x("act")).cuda()
        a2c_loss(pol32, torch.from_numpy(x("obs")).cuda(), act, torch.from_numpy(ret[h].reshape(-1)).cuda(), torch.from_numpy(x("val")).cuda(),
                 hp["ent_coef"], hp["vf_coef"]).backward()
        e32 = grad_errors([p.grad.cpu() for p in pol32.parameters()], [torch.from_numpy(g) for g in g64])
        grads.append(g64)
        bounds.append([grad_bound(float(np.abs(g).max())) + 4.0 * e for g, (e, _) in zip(g64, e32)])
        p_next, ms = clip_rmsprop_model(params[h], g64, ms, float(np.float32(lrs[h])), hp["max_grad_norm"], hp["alpha"], hp["epsilon"])
        params.append(p_next)
    # half 1 ran under the kernel's parameters after update 1, which lie within lr x (the update's gradient bound) + ulps of the float64 ones:
    # the towers' outputs may move by ~1e-5 more than float32 rounding of the same weights
    pols = [_with_params(r["template"], params[h], torch.float64).cpu() for h in range(n_up)]
    check_collection(r["env_id"], r["env_kwargs"], r["K"], SEED, buf, _np(r["obs"]), r["state"], pols, [h * T for h in range(n_up)],
                     _np(r["last_val"]), extra_tol=1.0 if n_up == 2 else 0.0)
    check_gae(buf, _np(r["last_val"]), _np(r["adv"]), ret, 1.0)
    # the last update's gradient
    h = n_up - 1
    kern = grad_errors([g.cpu() for g in r["grad"]], [torch.from_numpy(g) for g in grads[h]])
    print("  update %d: max|g - g64| / max|g64| kernel: " % (h + 1) + "  ".join("%s %.1e" % (n, e / max(s, 1e-30)) for n, (e, s) in zip(names, kern)))
    for k, name in enumerate(names):
        assert kern[k][0] <= bounds[h][k], (name, kern[k][0], bounds[h][k])
    # final parameters and slots: each update moves p by lr g_clipped / sqrt(ms + eps) with ms >= 0.99^2, so a clipped-gradient error e moves
    # it by at most 1.03 lr e; plus the float32 rounding of the parameter and of each step
    ep = [np.zeros(p.shape) for p in params[0]]
    ems = [np.zeros(p.shape) for p in params[0]]
    for u in range(n_up):
        gc, _, e = _clip_errors(grads[u], bounds[u])
        for k in range(len(ep)):
            ep[k] = ep[k] + 1.03 * lrs[u] * e[k]
            ems[k] = hp["alpha"] * ems[k] + (1 - hp["alpha"]) * e[k] * (2 * np.abs(gc[k]) + e[k])
    for k, name in enumerate(names):
        got = _np(r["after"][k]).astype(np.float64)
        tol = ep[k] + 3 * np.spacing(np.abs(params[-1][k]).astype(np.float32)).astype(np.float64)
        assert (np.abs(got - params[-1][k]) <= tol).all(), (name, np.abs(got - params[-1][k]).max())
        m = _np(r["ms"][k]).astype(np.float64)
        assert (np.abs(m - ms[k]) <= ems[k] + 4 * np.spacing(np.float32(1.0))).all(), (name, np.abs(m - ms[k]).max())
