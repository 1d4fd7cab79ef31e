"""
Mirror of the reference's training entry point ``python -m rl_baselines.train`` (rl_baselines/train.py:172-333) for the
algorithms this repo provides as consumers of the simulator: ``ppo2`` (rl_baselines/ppo2.py), ``a2c`` (rl_baselines/a2c.py), ``deepq``
(rl_baselines/deepq.py), ``sac`` (rl_baselines/sac.py), ``ddpg`` (rl_baselines/ddpg.py), ``trpo`` (rl_baselines/trpo.py) and ``random_agent`` (rl_baselines/random_agent.py:28-42).  Same flag names; ``--num-cpu`` is the number of envs in the
batch (per GPU when launched with ``torchrun --nproc-per-node N -m rl_baselines.train``: data-parallel PPO2, A2C or DQN, see rl_baselines/ppo2.py).
"""
import argparse
import os
import time

from environments.registry import registered_env

# rl_baselines/rl_algorithm/ppo2.py:25-36 (getOptParam): the hyper-parameters `--hyperparam name:value` may set, and their types
PPO2_OPT_PARAM = {"lam": float, "gamma": float, "max_grad_norm": float, "vf_coef": float, "learning_rate": float, "ent_coef": float,
                  "cliprange": float, "noptepochs": int, "n_steps": int}
# rl_baselines/rl_algorithm/a2c.py (A2CModel.getOptParam)
A2C_OPT_PARAM = {"n_steps": int, "vf_coef": float, "ent_coef": float, "max_grad_norm": float, "learning_rate": float, "epsilon": float,
                 "alpha": float, "gamma": float, "lr_schedule": str}
# rl_baselines/rl_algorithm/deepq.py:65-75 (DQNModel.getOptParam)
DQN_OPT_PARAM = {"learning_rate": float, "exploration_fraction": float, "exploration_final_eps": float, "train_freq": int, "learning_starts": int,
                 "target_network_update_freq": int, "gamma": float, "batch_size": int}
# rl_baselines/rl_algorithm/sac.py (SACModel.getOptParam)
SAC_OPT_PARAM = {"ent_coef": float, "learning_rate": float, "gradient_steps": int, "train_freq": int}
# rl_baselines/rl_algorithm/ddpg.py (DDPGModel.getOptParam)
DDPG_OPT_PARAM = {"reward_scale": float, "critic_l2_reg": float, "actor_lr": float, "critic_lr": float, "gamma": float, "nb_train_steps": int,
                  "nb_rollout_steps": int, "nb_eval_steps": int, "batch_size": int, "tau": float, "noise_action_sigma": float, "noise_action": str}
# rl_baselines/rl_algorithm/trpo.py (TRPOModel.getOptParam)
TRPO_OPT_PARAM = {"timesteps_per_batch": int, "max_kl": float, "cg_iters": int, "gamma": float, "lam": float, "entcoeff": float,
                  "cg_damping": float, "vf_stepsize": float, "vf_iters": int}
OPT_PARAM = {"ppo2": PPO2_OPT_PARAM, "a2c": A2C_OPT_PARAM, "deepq": DQN_OPT_PARAM, "sac": SAC_OPT_PARAM, "ddpg": DDPG_OPT_PARAM,
             "trpo": TRPO_OPT_PARAM}
LR_SCHEDULES = ['linear', 'constant', 'double_linear_con', 'middle_drop', 'double_middle_drop']


def parserHyperParam(pairs, opt_param=PPO2_OPT_PARAM):
    """``["name:value", ...]`` -> typed dict (train.py:321 + base_classes.py:62-80: unknown names are an AssertionError)."""
    parsed = {}
    for param in pairs:
        name, val = param.split(":")[0], param.split(":")[1]
        if name not in opt_param:
            raise AssertionError("Error: hyperparameter {} not in list of valid hyperparameters".format(name))
        parsed[name] = opt_param[name](val)
    if parsed.get("lr_schedule", LR_SCHEDULES[0]) not in LR_SCHEDULES:
        raise AssertionError("Error: lr_schedule {} not in {}".format(parsed["lr_schedule"], LR_SCHEDULES))
    return parsed


def main(argv=None):
    parser = argparse.ArgumentParser(description="Train script for RL algorithms")
    parser.add_argument('--algo', default='ppo2', choices=['ppo2', 'a2c', 'deepq', 'sac', 'ddpg', 'trpo', 'random_agent'], type=str)
    parser.add_argument('--env', type=str, help='environment ID', default='KukaButtonGymEnv-v0', choices=list(registered_env.keys()))
    parser.add_argument('--seed', type=int, default=0)
    parser.add_argument('--episode_window', type=int, default=40, help='Episode window for moving average plot (default: 40)')
    parser.add_argument('--num-stack', type=int, default=1, help='number of frames to stack (default: 1)')
    parser.add_argument('-joints', '--action-joints', action='store_true', default=False, help='set actions to the joints of the arm directly')
    parser.add_argument('--hyperparam', type=str, nargs='+', default=[], help='PPO2 / A2C / DQN / SAC / DDPG / TRPO hyper-parameters as name:value pairs')
    parser.add_argument('--lr-schedule', help='Learning rate schedule (a2c)', default='constant', choices=LR_SCHEDULES)
    parser.add_argument('--log-dir', default='/tmp/gym/', type=str)
    parser.add_argument('--num-timesteps', type=int, default=int(1e6))
    parser.add_argument('--srl-model', type=str, default='ground_truth', choices=['ground_truth'])
    parser.add_argument('--num-cpu', help='Number of envs in the lockstep batch', type=int, default=4096)
    parser.add_argument('--action-repeat', type=int, default=1)
    parser.add_argument('--shape-reward', action='store_true', default=False)
    parser.add_argument('-c', '--continuous-actions', action='store_true', default=False)
    parser.add_argument('-r', '--random-target', action='store_true', default=False)
    parser.add_argument('--device', type=int, default=0)
    # deepq's own flags (rl_algorithm/deepq.py:20-24); --dueling is accepted and has no effect: the deepq MlpPolicy is dueling either way
    parser.add_argument('--prioritized', type=int, default=1)
    parser.add_argument('--dueling', type=int, default=1)
    parser.add_argument('--buffer-size', type=int, default=None, help="Replay buffer size (default: 1000 for deepq, 50000 for sac, 100 for ddpg)")
    # ddpg's own flags (rl_algorithm/ddpg.py:22-37)
    parser.add_argument('--memory-limit', type=int, default=100000,
                        help='Accepted and has no effect, as in the reference, which never passes it to the model: the ring size is --buffer-size')
    parser.add_argument('--noise-action', type=str, default="ou", choices=["none", "normal", "ou"],
                        help='The type of action noise added to the output, can be gaussian or OrnsteinUhlenbeck (ddpg)')
    parser.add_argument('--noise-action-sigma', type=float, default=0.2, help='The variance of the action noise (ddpg)')
    parser.add_argument('--noise-param', action='store_true', default=False, help='Enable parameter noise (ddpg: not supported, refused)')
    parser.add_argument('--noise-param-sigma', type=float, default=0.2, help='The variance of the parameter noise (ddpg: not supported)')
    parser.add_argument('--batch-size', type=int, default=64, help='The batch size used for training (ddpg)')
    args, _ = parser.parse_known_args(argv)
    # sanity checks of the reference (train.py:221-224,265-266)
    assert args.episode_window >= 1, "Error: --episode_window cannot be less than 1"
    assert args.num_timesteps >= 1, "Error: --num-timesteps cannot be less than 1"
    assert args.num_stack >= 1, "Error: --num-stack cannot be less than 1"
    assert args.action_repeat >= 1, "Error: --action-repeat cannot be less than 1"
    if args.action_joints and not args.continuous_actions:
        raise ValueError("The joints action space is continuous only: use '-joints' together with '-c' (kuka_button_gym_env.py:149-161)")
    if args.algo == "deepq" and args.continuous_actions:       # train.py:260-262
        from rl_baselines.deepq import CONTINUOUS_ERROR
        raise ValueError(CONTINUOUS_ERROR)
    if args.algo == "sac" and not args.continuous_actions:    # train.py:257-259
        from rl_baselines.sac import DISCRETE_ERROR
        raise ValueError(DISCRETE_ERROR)
    if args.algo == "ddpg" and not args.continuous_actions:   # train.py:257-259
        from rl_baselines.ddpg import DISCRETE_ERROR
        raise ValueError(DISCRETE_ERROR)
    hyperparams = parserHyperParam(args.hyperparam, OPT_PARAM.get(args.algo, PPO2_OPT_PARAM))
    if args.algo == "a2c":
        hyperparams = dict(dict(lr_schedule=args.lr_schedule), **hyperparams)
    if args.algo == "deepq":
        hyperparams = dict(dict(buffer_size=args.buffer_size or int(1e3), prioritized_replay=bool(args.prioritized)), **hyperparams)
    if args.algo == "sac":
        hyperparams = dict(dict(buffer_size=args.buffer_size or 50000), **hyperparams)
    if args.algo == "ddpg":                                   # rl_algorithm/ddpg.py:111-119,149-153: --hyperparam wins over the noise flags
        from rl_baselines.ddpg import MEMORY_LIMIT
        hyperparams = dict(dict(buffer_size=args.buffer_size or MEMORY_LIMIT, batch_size=args.batch_size, noise_action=args.noise_action,
                                noise_action_sigma=args.noise_action_sigma), **hyperparams)
    env_kwargs = dict(is_discrete=not args.continuous_actions, action_repeat=args.action_repeat, random_target=args.random_target,
                      shape_reward=args.shape_reward, srl_model=args.srl_model)
    if args.action_joints:
        env_kwargs["action_joints"] = True
    log_dir = os.path.join(args.log_dir, args.env, args.srl_model, args.algo, time.strftime("%y-%m-%d_%Hh%M_%S"))
    num_timesteps = int(1.1 * args.num_timesteps)      # the reference trains 10 % longer (train.py:319)
    if args.algo in ("ppo2", "a2c", "deepq", "sac", "ddpg", "trpo"):
        if args.algo == "ppo2":
            from rl_baselines.ppo2 import train
        elif args.algo == "a2c":
            from rl_baselines.a2c import train
        elif args.algo == "sac":
            from rl_baselines.sac import train
        elif args.algo == "ddpg":
            from rl_baselines.ddpg import train
        elif args.algo == "trpo":
            from rl_baselines.trpo import train
        else:
            from rl_baselines.deepq import train
        from srl_sim.distributed import rank_world
        rank, world, local_rank = rank_world()
        device = args.device
        if world > 1:      # torchrun: one process per GPU, --num-cpu envs on EACH rank, gradients averaged over NCCL
            import torch
            import torch.distributed as dist
            device = local_rank
            torch.cuda.set_device(device)
            if not dist.is_initialized():
                dist.init_process_group("nccl", device_id=torch.device("cuda", device))
        extra = dict(noise_param=args.noise_param) if args.algo == "ddpg" else {}
        try:
            return train(args.env, args.num_cpu, num_timesteps, seed=args.seed, env_kwargs=env_kwargs, log_dir=log_dir, device=device,
                         hyperparams=hyperparams, episode_window=args.episode_window, num_stack=args.num_stack, **extra)
        finally:
            if world > 1 and dist.is_initialized():
                dist.destroy_process_group()
    from rl_baselines.random_agent import train
    return train(args.env, args.num_cpu, num_timesteps, seed=args.seed, env_kwargs=env_kwargs, num_stack=args.num_stack)


if __name__ == '__main__':
    main()
