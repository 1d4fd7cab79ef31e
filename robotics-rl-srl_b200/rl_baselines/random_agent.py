"""
Mirror of rl_baselines/random_agent.py:28-42 -- the reference's own throughput harness: sample actions, step the VecEnv,
print "{steps} steps - {FPS}" every 500 updates.
"""
import time

from srl_sim.vec_env import BatchedSRLVecEnv


def train(env_id, num_cpu, num_timesteps, seed=0, env_kwargs=None, device=None, verbose=1, num_stack=1):
    env = BatchedSRLVecEnv(env_id, num_cpu, seed=seed, device=device, **(env_kwargs or {}))
    if num_stack > 1:                  # the reference's createEnvs stacks for every algorithm (rl_baselines/utils.py:222)
        from rl_baselines.utils import VecFrameStack
        env = VecFrameStack(env, num_stack)
    env.action_space.seed(seed)
    env.reset()
    num_updates = int(num_timesteps) // num_cpu
    start_time = time.time()
    fps = 0.0
    for step in range(num_updates):
        actions = [env.action_space.sample() for _ in range(num_cpu)]
        env.step(actions)
        if (step + 1) % 500 == 0 or step + 1 == num_updates:
            total_steps = (step + 1) * num_cpu
            fps = total_steps / (time.time() - start_time)
            if verbose:
                print("{} steps - {:.2f} FPS".format(total_steps, fps))
    env.close()
    return fps
