"""
Mirror of the reference's replay entry point ``python -m replay.enjoy_baselines --log-dir <trained agent>``
(replay/enjoy_baselines.py:45-63 arguments, :66-118 config loading, :151-333 the enjoy loop) for the agents this repo can
train: it reloads ``args.json`` / ``env_globals.json`` / ``<algo>_model.pt`` written by ``rl_baselines.ppo2.train`` or ``rl_baselines.a2c.train``
(the same MlpPolicy), ``rl_baselines.deepq.train`` (the dueling Q network, always greedy: stable-baselines' DQN.predict) or ``rl_baselines.sac.train``
(the squashed Gaussian actor: ``tanh(mu)`` with ``--deterministic``, a sample otherwise), rebuilds the
env batch with the training-time keyword arguments and the saved observation filter (``load_path_normalise``, :145), runs the
policy for ``--num-timesteps`` steps and reports ``"<n> episodes - Mean reward: <r>"`` like the reference (:330-333).
Rendering / plotting flags are accepted and ignored (image observations are out of scope, DESIGN.md section 8).
"""
import argparse
import json
import os

import numpy as np
import torch

from rl_baselines.ppo2 import MlpPolicy
from srl_sim.vec_env import BatchedSRLVecEnv


def parseArguments(argv=None):
    parser = argparse.ArgumentParser(description="Enjoy trained agent")
    parser.add_argument('--seed', type=int, default=0, help='random seed (default: 0)')
    parser.add_argument('--num-cpu', help='Number of envs in the batch', type=int, default=1)
    parser.add_argument('--log-dir', help='folder with the saved agent model', type=str, required=True)
    parser.add_argument('--num-timesteps', type=int, default=int(1e4))
    parser.add_argument('--render', action='store_true', default=False, help='accepted, ignored')
    parser.add_argument('--shape-reward', action='store_true', default=False)
    parser.add_argument('--plotting', action='store_true', default=False, help='accepted, ignored')
    parser.add_argument('--action-proba', action='store_true', default=False, help='accepted, ignored')
    parser.add_argument('--deterministic', action='store_true', default=False, help='greedy actions instead of sampling')
    parser.add_argument('--device', type=int, default=0)
    return parser.parse_args(argv)


def loadConfigAndSetup(load_args):
    """(train_args, load_path, env_kwargs) of a finished training run (enjoy_baselines.py:66-118)."""
    log_dir = load_args.log_dir
    with open(os.path.join(log_dir, "env_globals.json")) as f:
        env_globals = json.load(f)
    with open(os.path.join(log_dir, "args.json")) as f:
        train_args = json.load(f)
    algo = train_args.get("algo", "ppo2")
    if algo not in ("ppo2", "a2c", "deepq", "sac"):
        raise ValueError(algo + " is not supported for replay")
    env_kwargs = dict(env_globals)
    env_kwargs["shape_reward"] = load_args.shape_reward            # reward sparse or shaped: chosen at replay time (:88)
    env_kwargs["srl_model"] = train_args.get("srl_model", "ground_truth")
    return train_args, os.path.join(log_dir, algo + "_model.pt"), env_kwargs


def main(argv=None):
    load_args = parseArguments(argv)
    train_args, load_path, env_kwargs = loadConfigAndSetup(load_args)
    torch.manual_seed(load_args.seed)
    env = BatchedSRLVecEnv(train_args["env"], load_args.num_cpu, seed=load_args.seed, device=load_args.device, **env_kwargs)
    on_gpu = env.backend.on_gpu
    dev = env.backend.torch_device if on_gpu else torch.device("cpu")   # device -1: the CPU oracle a test installs (numpy buffers)
    as_tensor = (lambda x: x) if on_gpu else torch.from_numpy
    D = env.observation_space.shape[0]
    K = int(train_args.get("num_stack", 1))                       # VecFrameStack of the training run (:140)
    W = K * D
    deepq, sac = train_args.get("algo") == "deepq", train_args.get("algo") == "sac"
    if sac:
        from rl_baselines.sac import SACNets
        policy = SACNets(W, env.action_space.shape[0]).to(dev)
    elif deepq:
        from rl_baselines.deepq import DuelingQ
        policy = DuelingQ(W, env.action_space.n).to(dev)
    else:
        policy = (MlpPolicy(W, n_actions=env.action_space.n) if env.is_discrete else MlpPolicy(W, action_dim=env.action_space.shape[0])).to(dev)
    saved = torch.load(load_path, map_location=dev)
    policy.load_state_dict(saved["policy"])
    mean, var = saved["obs_mean"].float().to(dev), saved["obs_var"].float().to(dev)

    def normalise(o):                                              # VecNormalize in test mode: frozen statistics, clip +-10
        return torch.clamp((o - mean) / torch.sqrt(var + 1e-8), -10.0, 10.0)

    env.sim.reset(obs_out=env._obs, stream=env.backend.stream())
    stack = torch.zeros((load_args.num_cpu, W), device=dev)       # the trainer's frame stack: oldest frame first, zeroed where an episode ended
    stack[:, W - D:].copy_(as_tensor(env._obs))
    obs = normalise(stack.clone())
    n_done, returns = 0, []
    with torch.no_grad():
        for _ in range(load_args.num_timesteps):
            if sac:
                a = policy.act(obs, deterministic=load_args.deterministic)
            elif deepq:
                a = policy(obs).argmax(-1)
            else:
                dist = policy.dist(obs)
                if load_args.deterministic:
                    a = dist.probs.argmax(-1) if env.is_discrete else dist.mean
                else:
                    a = dist.sample()
            act = a.to(torch.int32) if env.is_discrete else torch.clamp(a, -1, 1).contiguous()
            o, _, d, ep_ret, _ = (as_tensor(x) for x in env.step_tensors(act))
            if bool(d.any()):
                returns.extend(ep_ret[d.bool()].tolist())
                if len(returns) - n_done > 1:                      # the reference prints whenever more than one episode ended (:327-330)
                    n_done = len(returns)
                    print("{} episodes - Mean reward: {:.2f}".format(n_done, float(np.mean(returns))))
            stack.copy_(torch.where(d.bool()[:, None], 0.0, torch.roll(stack, -D, 1)))
            stack[:, W - D:].copy_(o)
            obs = normalise(stack.clone())
    n_done = len(returns)
    mean_reward = float(np.mean(returns)) if returns else float("nan")
    print("{} episodes - Mean reward: {:.2f}".format(n_done, mean_reward))
    env.close()
    return n_done, mean_reward


if __name__ == '__main__':
    main()
