"""
``BatchedSRLVecEnv`` -- a stable-baselines-style ``VecEnv`` over ONE lockstep batch of simulated envs.

It takes the place of the ``SubprocVecEnv`` / ``DummyVecEnv`` the reference builds in
``rl_baselines/utils.py:194-229`` (``createEnvs``): instead of one OS process per env exchanging pickled
(obs, reward, done, info) tuples over pipes, all ``num_envs`` envs live in structure-of-arrays HBM and one
kernel launch steps them.  Semantics kept from stable-baselines 2.5 (SURVEY.md Appendix B.3):

* ``reset() -> obs[N, D]``; ``step_async(actions)`` / ``step_wait()`` / ``step(actions)``
  ``-> (obs[N, D], rewards[N], dones[N], infos[N])``;
* an env that finishes is reset immediately and the returned observation is the post-reset one;
* ``infos[i]['episode'] = {'r': return, 'l': length, 't': wall time}`` on done (``bench.Monitor``, environments/utils.py:53-54).

numpy in / numpy out by default; ``step_tensors`` / ``rollout_tensors`` keep everything on the GPU (zero copies) for a
GPU-resident policy.
"""
import time

import numpy as np

from . import _abi, spaces
from .backend import default_backend

_KUKA_IDS = ("KukaButtonGymEnv-v0", "KukaRandButtonGymEnv-v0", "KukaMovingButtonGymEnv-v0", "Kuka2ButtonGymEnv-v0")
_OBS_DIM = {"MobileRobot1DGymEnv-v0": 1}
_N_ACTIONS = {"MobileRobot1DGymEnv-v0": 2, "MobileRobotGymEnv-v0": 4, "MobileRobot2TargetGymEnv-v0": 4,
              "MobileRobotLineTargetGymEnv-v0": 4, "KukaButtonGymEnv-v0": 6, "KukaRandButtonGymEnv-v0": 6, "KukaMovingButtonGymEnv-v0": 6,
              "Kuka2ButtonGymEnv-v0": 6}


class BatchedSRLVecEnv(object):
    """
    :param env_id: (str) one of the ids of ``environments.registry.registered_env``
    :param num_envs: (int) envs in this process / on this GPU
    :param seed: (int) base seed; env ``i`` uses the stream of global index ``global_env_offset + i``
    :param device: (int) CUDA ordinal (default 0)
    :param global_env_offset: (int) index of local env 0 in the global batch (rank * num_envs under torchrun)
    :param log_dir: (str) if given, every finished episode is appended to ``<log_dir>/<global_env_offset>.monitor.csv``
        (``bench.Monitor`` format; the reference writes one such file per env process, environments/utils.py:53-54)
    :param env_kwargs: the reference's env keyword arguments (is_discrete, random_target, shape_reward, force_down,
        action_repeat, max_distance, srl_model, ...); unknown ones are ignored like the reference's ``**_``
    """

    def __init__(self, env_id, num_envs, seed=0, device=None, global_env_offset=0, log_dir=None, **env_kwargs):
        if env_id not in _abi.ENV_KINDS:
            raise KeyError("unknown env id %r" % env_id)
        srl_model = env_kwargs.pop("srl_model", "ground_truth")
        kuka_state_models = ("joints", "joints_position") if env_id.startswith("Kuka") else ()
        if srl_model not in ("ground_truth", "raw_pixels") and srl_model not in kuka_state_models:
            raise NotImplementedError("BatchedSRLVecEnv provides ground_truth%s states and raw_pixels frames (got srl_model=%r; learned SRL models are out of scope)"
                                      % ("".join(" / " + m for m in kuka_state_models), srl_model))
        # raw_pixels: one rendered frame per env and camera (srl_sim/render.py; multi_view / fpv stack a second camera on the channels)
        self._cams = None
        self._fpv_cams = None
        if srl_model == "raw_pixels":
            from . import render as _render
            if env_id.startswith("Kuka"):
                self._cams = [_render.KUKA_CAMERA] + ([_render.KUKA_CAMERA_2] if env_kwargs.get("multi_view", False) else [])
            else:
                self._cams = [dict(_render.MOBILE_CAMERA, target=(2, 0, 0) if env_id == "MobileRobot1DGymEnv-v0" else (2, 2, 0))]
                if env_kwargs.get("fpv", False):
                    # each env's first-person camera follows its robot (mobile_robot_env.py:316-332): one camera per env, built once here
                    # and finished from the robot positions on the device at every render
                    self._fpv_cams = _render.camera_array([_render.MOBILE_FPV_FOLLOW] * int(num_envs))
        self.distractors = bool(env_kwargs.get("distractors", False))
        if self.distractors and env_id != "KukaRandButtonGymEnv-v0":
            raise ValueError("distractors=True is only available for KukaRandButtonGymEnv-v0 (got %r)" % env_id)
        self.srl_model = srl_model
        self.env_id = env_id
        self.num_envs = int(num_envs)
        self.backend = default_backend(device)
        cfg = dict(is_discrete=env_kwargs.get("is_discrete", True), random_target=env_kwargs.get("random_target", False),
                   shape_reward=env_kwargs.get("shape_reward", False), force_down=env_kwargs.get("force_down", True),
                   action_repeat=env_kwargs.get("action_repeat", 1), action_joints=env_kwargs.get("action_joints", False),
                   global_env_offset=global_env_offset)
        blob = None
        if env_id in _KUKA_IDS:
            from .model import load_kuka_scene
            blob = load_kuka_scene().blob
            two = env_id == "Kuka2ButtonGymEnv-v0"     # its constructor defaults differ (kuka_2button_gym_env.py:30-31)
            cfg["max_distance"] = env_kwargs.get("max_distance", 2.0 if two else 0.8)
            cfg["force_down"] = env_kwargs.get("force_down", not two)
        for k in ("max_steps", "envs_per_warp", "solver_iterations", "prefetch_resets"):
            if k in env_kwargs:
                cfg[k] = env_kwargs[k]
        self.sim = self.backend.make_sim(env_id, self.num_envs, seed=seed, model_blob=blob, **cfg)
        if self.distractors:
            # kuka_rand_button_gym_env.py:58-68: random objects around the button and a kicked sphere (one-way coupled: the arm's outputs do not
            # change); srl_sim_render draws them, so raw_pixels observations and render_tensors() show them
            from .model import distractor_blob
            self.sim.set_distractors(distractor_blob())
        self.is_discrete = bool(cfg["is_discrete"])
        D = self.sim.obs_dim
        # Kuka `joints` / `joints_position` states (kuka_button_gym_env.py:175-189): the 14 stored joint positions are the
        # INITIAL vector -- the reference never updates `_kuka.joint_positions` (kuka.py:65-66) -- so they are a constant
        self._joints = None
        if srl_model in ("joints", "joints_position"):
            from .model import KUKA_INIT_JOINT_POSITIONS
            self._joints = np.tile(np.asarray(KUKA_INIT_JOINT_POSITIONS, np.float32), (self.num_envs, 1))
        if srl_model == "raw_pixels":
            from .render import RENDER_HEIGHT, RENDER_WIDTH
            n_cams = len(self._cams) + (self._fpv_cams is not None)
            self.observation_space = spaces.Box(low=0, high=255, shape=(RENDER_HEIGHT, RENDER_WIDTH, 3 * n_cams), dtype=np.uint8)
        else:
            out_dim = {"ground_truth": D, "joints": 14, "joints_position": D + 14}[srl_model]
            self.observation_space = spaces.Box(low=-np.inf, high=np.inf, shape=(out_dim,), dtype=np.float32)
        self._monitor = None
        if log_dir is not None:
            from .monitor import MonitorWriter
            import os
            self._monitor = MonitorWriter(os.path.join(log_dir, str(global_env_offset)), env_id=env_id)
        if self.is_discrete:
            self.action_space = spaces.Discrete(_N_ACTIONS[env_id])
        else:
            self.action_space = spaces.Box(low=-1, high=1, shape=(self.sim.action_dim,), dtype=np.float32)
        be = self.backend
        n = self.num_envs
        self._obs = be.zeros((n, D), np.float32)
        self._rew = be.zeros((n,), np.float32)
        self._done = be.zeros((n,), np.uint8)
        self._ep_ret = be.zeros((n,), np.float32)
        self._ep_len = be.zeros((n,), np.int32)
        self._actions = None
        self._t0 = time.time()
        self.closed = False

    # ---- VecEnv API (numpy) --------------------------------------------------------------------------
    def render_tensors(self):
        """The current frame of every env, ``uint8 [N, H, W, 3 * cameras]`` in the backend's memory (a CUDA tensor on a GPU); with ``fpv``
        the first-person frames are the last three channels."""
        from .render import KUKA_CAMERA, MOBILE_CAMERA, render_batch, render_cameras
        cams = self._cams or ([KUKA_CAMERA] if self.env_id.startswith("Kuka") else [MOBILE_CAMERA])
        frames = render_batch(self.sim, self.backend, cams)
        if self._fpv_cams is None:
            return frames
        fpv = render_cameras(self.sim, self.backend, self._fpv_cams, follow_robot=True)
        if self.backend.on_gpu:
            return self.backend.torch.cat([frames, fpv], dim=3)
        return np.concatenate([frames, fpv], axis=3)

    def _state(self, obs):
        """ground-truth observation [N, D] -> the configured state (getSRLState), or the rendered frames (raw_pixels)."""
        if self.srl_model == "raw_pixels":
            return self.backend.to_host(self.render_tensors()).copy()
        if self._joints is None:
            return obs
        return self._joints.copy() if self.srl_model == "joints" else np.concatenate([obs, self._joints], axis=1)

    def reset(self):
        self.sim.reset(obs_out=self._obs, stream=self.backend.stream())
        return self._state(self.backend.to_host(self._obs).copy())

    def step_async(self, actions):
        if self.is_discrete:
            a = np.asarray([-1 if x is None else x for x in actions] if isinstance(actions, (list, tuple)) else actions, dtype=np.int32)
            a = a.reshape(self.num_envs)
        else:
            a = np.asarray(actions, dtype=np.float32).reshape(self.num_envs, self.sim.action_dim)
        self._actions = self.backend.from_host(a)

    def step_wait(self):
        be = self.backend
        self.sim.step(self._actions, None, self._obs, self._rew, self._done, self._ep_ret, self._ep_len, stream=be.stream())
        obs = be.to_host(self._obs).copy()
        rew = be.to_host(self._rew).copy()
        done = be.to_host(self._done).astype(bool)
        infos = [{} for _ in range(self.num_envs)]
        if done.any():
            ep_ret, ep_len = be.to_host(self._ep_ret), be.to_host(self._ep_len)
            t = round(time.time() - self._t0, 6)
            for i in np.nonzero(done)[0]:
                if self._monitor is not None:
                    infos[i]["episode"] = self._monitor.write_episode(ep_ret[i], ep_len[i])
                else:
                    infos[i]["episode"] = {"r": round(float(ep_ret[i]), 6), "l": int(ep_len[i]), "t": t}
        return self._state(obs), rew, done, infos

    def step(self, actions):
        self.step_async(actions)
        return self.step_wait()

    def close(self):
        if not self.closed:
            self.sim.close()
            if self._monitor is not None:
                self._monitor.close()
            self.closed = True

    def seed(self, seed=None):
        raise NotImplementedError("the batch is seeded at construction (counter-based streams keyed by env index)")

    def get_images(self):
        """VecEnv.get_images: one RGB frame per env (numpy)."""
        return list(self.backend.to_host(self.render_tensors()))

    def render(self, mode="human"):
        raise NotImplementedError("image observations are out of scope of the batched simulator")

    # ---- zero-copy GPU API ---------------------------------------------------------------------------
    def step_tensors(self, actions, noise=None):
        """``actions``: torch CUDA tensor int32[N] / float32[N, A]; returns CUDA tensors (views of internal buffers)."""
        self.sim.step(actions, noise, self._obs, self._rew, self._done, self._ep_ret, self._ep_len, stream=self.backend.stream())
        return self._obs, self._rew, self._done, self._ep_ret, self._ep_len

    def rollout_tensors(self, T, actions=None, noise=None, out=None):
        """T fused steps in one launch.  ``actions``: CUDA int32[T, N] / float32[T, N, A] or None (random agent)."""
        be, n, D = self.backend, self.num_envs, self.sim.obs_dim
        if out is None:
            out = dict(obs=be.empty((T, n, D), np.float32), rew=be.empty((T, n), np.float32), done=be.empty((T, n), np.uint8),
                       ep_ret=be.zeros((T, n), np.float32), ep_len=be.zeros((T, n), np.int32))
        self.sim.rollout(T, actions, noise, out["obs"], out["rew"], out["done"], out["ep_ret"], out["ep_len"], stream=be.stream())
        return out
