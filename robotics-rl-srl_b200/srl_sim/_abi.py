"""
ctypes binding of the C-ABI declared in ``include/srl_sim.h``.

The product library is ``csrc/libsrl_sim_b200.so`` (hand-written sm_90a CUDA).  There is no
CPU fallback: if the library is missing or cannot be loaded, :func:`load_cuda_library` raises.
``SimLibrary`` itself is path-agnostic, so the test-suite can drive the CPU oracle (which exports
the same symbols) through the very same binding.

Reference interface mirrored: the per-process env objects behind
``environments/utils.py:36-57`` (``makeEnv``) and ``rl_baselines/utils.py:194-229`` (``createEnvs``).
"""
import ctypes
import os
from ctypes import (POINTER, Structure, byref, c_char_p, c_double, c_float, c_int, c_int32,
                    c_size_t, c_uint8, c_uint32, c_uint64, c_void_p)

import numpy as np

ABI_VERSION = 1

# environments/registry.py:42-49
ENV_KINDS = {
    "KukaButtonGymEnv-v0": 0,
    "KukaRandButtonGymEnv-v0": 1,
    "Kuka2ButtonGymEnv-v0": 2,
    "KukaMovingButtonGymEnv-v0": 3,
    "MobileRobotGymEnv-v0": 4,
    "MobileRobot2TargetGymEnv-v0": 5,
    "MobileRobot1DGymEnv-v0": 6,
    "MobileRobotLineTargetGymEnv-v0": 7,
}

# enum srl_state_field
F_ROBOT_POS, F_TARGET_POS, F_STEP_COUNTER, F_JOINT_POS, F_JOINT_VEL, F_EE_CMD, F_EE_POS, \
    F_BUTTON_GLIDER, F_COUNTERS, F_EPISODE_STATS, F_BUTTON_BASE, F_TWO_BUTTON, F_NEXT_RECORD, F_DISTRACTORS, F_DISTRACTOR_TOUCH = range(15)

_FIELD_SPEC = {
    F_ROBOT_POS: (np.float64, 3), F_TARGET_POS: (np.float64, 3), F_STEP_COUNTER: (np.int32, 1),
    F_JOINT_POS: (np.float64, 12), F_JOINT_VEL: (np.float64, 12), F_EE_CMD: (np.float64, 3),
    F_EE_POS: (np.float64, 3), F_BUTTON_GLIDER: (np.float64, 2), F_COUNTERS: (np.int32, 4),
    F_EPISODE_STATS: (np.float64, 2), F_BUTTON_BASE: (np.float64, 3), F_TWO_BUTTON: (np.float64, 8), F_NEXT_RECORD: (np.int32, 3),
    F_DISTRACTORS: (np.float64, 11 * 9), F_DISTRACTOR_TOUCH: (np.int32, 2),
}

MOBILE_RESET_DRAWS = 6
KUKA_RESET_DRAWS = 18
KUKA_DISTRACTOR_RESET_DRAWS = 48   # with srl_sim_set_distractors: + 10 placements (x, y) + 10 object types


class SrlCfg(Structure):
    """struct srl_cfg (include/srl_sim.h)."""
    _fields_ = [
        ("struct_size", c_uint32),
        ("is_discrete", c_int32),
        ("random_target", c_int32),
        ("force_down", c_int32),
        ("shape_reward", c_int32),
        ("action_joints", c_int32),
        ("action_repeat", c_int32),
        ("max_steps", c_int32),
        ("solver_iterations", c_int32),
        ("envs_per_warp", c_int32),
        ("no_auto_reset", c_int32),
        ("max_distance", c_float),
        ("timestep", c_float),
        ("prefetch_resets", c_uint32),
        ("global_env_offset", c_uint64),
    ]


class SimError(RuntimeError):
    pass


_EXPORTS = [
    # name, restype, argtypes
    ("srl_sim_abi_version", c_int, []),
    ("srl_sim_create", c_int, [POINTER(c_void_p), c_int, c_int, c_int, POINTER(SrlCfg), c_void_p, c_size_t, c_uint64]),
    ("srl_sim_reset", c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    ("srl_sim_step", c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    ("srl_sim_rollout", c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    ("srl_sim_rollout_host", c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    ("srl_sim_prefetch_resets", c_int, [c_void_p, c_void_p]),
    ("srl_sim_render", c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    ("srl_sim_render_cameras", c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    ("srl_sim_set_distractors", c_int, [c_void_p, c_void_p, c_size_t]),
    ("srl_sim_get_state", c_int, [c_void_p, c_int, c_void_p, c_size_t]),
    ("srl_sim_set_state", c_int, [c_void_p, c_int, c_void_p, c_size_t]),
    ("srl_sim_launch_count", c_uint64, [c_void_p]),
    ("srl_sim_last_kernel_ms", c_float, [c_void_p]),
    ("srl_sim_num_envs", c_int, [c_void_p]),
    ("srl_sim_obs_dim", c_int, [c_void_p]),
    ("srl_sim_action_dim", c_int, [c_void_p]),
    ("srl_sim_last_error", c_char_p, []),
    ("srl_sim_destroy", None, [c_void_p]),
]

EXPORTED_SYMBOLS = [e[0] for e in _EXPORTS]   # everything include/srl_sim.h declares


def _ptr(x):
    """Raw address of a numpy array / torch tensor / int / None."""
    if x is None:
        return None
    if isinstance(x, int):
        return x
    if isinstance(x, np.ndarray):
        if not x.flags["C_CONTIGUOUS"]:
            raise ValueError("buffer must be C-contiguous")
        return x.ctypes.data
    if hasattr(x, "data_ptr"):  # torch tensor
        if not x.is_contiguous():
            raise ValueError("tensor must be contiguous")
        return x.data_ptr()
    raise TypeError("unsupported buffer type %r" % type(x))


class SimLibrary(object):
    """A loaded shared library exporting the srl_sim C-ABI."""

    def __init__(self, path):
        if not os.path.isfile(path):
            raise SimError("srl_sim library not found: %s" % path)
        self.path = os.path.abspath(path)
        self.lib = ctypes.CDLL(self.path)
        for name, restype, argtypes in _EXPORTS:
            try:
                fn = getattr(self.lib, name)
            except AttributeError:
                raise SimError("%s does not export %s" % (self.path, name))
            fn.restype = restype
            fn.argtypes = argtypes
        v = self.lib.srl_sim_abi_version()
        if v != ABI_VERSION:
            raise SimError("ABI version mismatch: library %d, binding %d" % (v, ABI_VERSION))

    def last_error(self):
        msg = self.lib.srl_sim_last_error()
        return msg.decode("utf-8", "replace") if msg else ""

    def check(self, rc, what):
        if rc != 0:
            msg = self.last_error()
            # the reference raises ValueError for unsupported action modes
            # (mobile_robot_1D_env.py:43,118; mobile_robot_2target_env.py:128)
            if rc == 2:
                raise ValueError(msg)
            raise SimError("%s failed (rc=%d): %s" % (what, rc, msg))


class Sim(object):
    """One ``srl_sim`` handle: ``num_envs`` environments of one kind, stepped in lockstep."""

    def __init__(self, library, env_kind, num_envs, device, seed=0, model_blob=None, **cfg):
        self.library = library
        self._lib = library.lib
        self.handle = c_void_p()
        if isinstance(env_kind, str):
            env_kind = ENV_KINDS[env_kind]
        self.env_kind = env_kind
        c = SrlCfg()
        c.struct_size = ctypes.sizeof(SrlCfg)
        c.is_discrete = int(cfg.pop("is_discrete", True))
        c.random_target = int(cfg.pop("random_target", False))
        c.force_down = int(cfg.pop("force_down", True))
        c.shape_reward = int(cfg.pop("shape_reward", False))
        c.action_joints = int(cfg.pop("action_joints", False))
        c.action_repeat = int(cfg.pop("action_repeat", 1))
        c.max_steps = int(cfg.pop("max_steps", 0))
        c.solver_iterations = int(cfg.pop("solver_iterations", 0))
        c.envs_per_warp = int(cfg.pop("envs_per_warp", 0))
        c.no_auto_reset = int(cfg.pop("no_auto_reset", False))
        c.max_distance = float(cfg.pop("max_distance", 0.8))
        c.timestep = float(cfg.pop("timestep", 0.0))
        c.prefetch_resets = int(bool(cfg.pop("prefetch_resets", False)))
        c.global_env_offset = int(cfg.pop("global_env_offset", 0))
        if cfg:
            raise TypeError("unknown cfg keys: %s" % sorted(cfg))
        self.cfg = c
        blob_ptr, blob_len = None, 0
        if model_blob is not None:
            self._blob = np.ascontiguousarray(model_blob)
            blob_ptr, blob_len = self._blob.ctypes.data, self._blob.nbytes
        rc = self._lib.srl_sim_create(byref(self.handle), env_kind, int(num_envs), int(device), byref(c),
                                      blob_ptr, blob_len, int(seed) & 0xFFFFFFFFFFFFFFFF)
        library.check(rc, "srl_sim_create")
        self.num_envs = self._lib.srl_sim_num_envs(self.handle)
        self.obs_dim = self._lib.srl_sim_obs_dim(self.handle)
        self.action_dim = self._lib.srl_sim_action_dim(self.handle)
        self.is_discrete = bool(c.is_discrete)
        self.device = device

    # -- lifecycle -------------------------------------------------------------------------
    def close(self):
        if self.handle:
            self._lib.srl_sim_destroy(self.handle)
            self.handle = c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- stepping (raw pointers; callers pass numpy arrays for the oracle, torch CUDA tensors for
    #    the CUDA library) ------------------------------------------------------------------
    def reset(self, mask=None, reset_draws=None, obs_out=None, stream=None):
        rc = self._lib.srl_sim_reset(self.handle, _ptr(mask), _ptr(reset_draws), _ptr(obs_out), stream)
        self.library.check(rc, "srl_sim_reset")

    def step(self, actions, noise=None, obs_out=None, rew_out=None, done_out=None, ep_ret_out=None,
             ep_len_out=None, stream=None):
        rc = self._lib.srl_sim_step(self.handle, _ptr(actions), _ptr(noise), _ptr(obs_out), _ptr(rew_out),
                                    _ptr(done_out), _ptr(ep_ret_out), _ptr(ep_len_out), stream)
        self.library.check(rc, "srl_sim_step")

    def rollout(self, T, actions=None, noise=None, obs_out=None, rew_out=None, done_out=None,
                ep_ret_out=None, ep_len_out=None, stream=None):
        rc = self._lib.srl_sim_rollout(self.handle, int(T), _ptr(actions), _ptr(noise), _ptr(obs_out),
                                       _ptr(rew_out), _ptr(done_out), _ptr(ep_ret_out), _ptr(ep_len_out), stream)
        self.library.check(rc, "srl_sim_rollout")

    def rollout_host(self, T, actions=None, noise=None, obs_out=None, rew_out=None, done_out=None):
        rc = self._lib.srl_sim_rollout_host(self.handle, int(T), _ptr(actions), _ptr(noise), _ptr(obs_out),
                                            _ptr(rew_out), _ptr(done_out))
        self.library.check(rc, "srl_sim_rollout_host")

    def prefetch_resets(self, stream=None):
        """Bulk fill of the next-episode records (handles created with ``prefetch_resets=True``; a no-op otherwise).  In steady state
        the helper slots of every step / rollout launch keep the records up; call this once after a reset of all envs."""
        rc = self._lib.srl_sim_prefetch_resets(self.handle, stream)
        self.library.check(rc, "srl_sim_prefetch_resets")

    def render(self, cam, width, height, rgb_out, stream=None):
        """One ``width`` x ``height`` RGB frame per env into ``rgb_out`` (u8[N, H, W, 3]); ``cam`` is an ``srl_sim.render.SrlCamera``."""
        rc = self._lib.srl_sim_render(self.handle, ctypes.byref(cam), int(width), int(height), _ptr(rgb_out), stream)
        self.library.check(rc, "srl_sim_render")

    def render_cameras(self, cams, follow_robot, width, height, rgb_out, stream=None):
        """One frame per env through its own camera: ``cams`` is a ctypes array of ``num_envs`` ``srl_sim.render.SrlCamera``; with
        ``follow_robot`` (MobileRobot) each target's x and y are offsets from that env's robot position."""
        if cams is not None and len(cams) != self.num_envs:
            raise ValueError("render_cameras: %d cameras for %d envs" % (len(cams), self.num_envs))
        rc = self._lib.srl_sim_render_cameras(self.handle, cams, int(bool(follow_robot)), int(width), int(height), _ptr(rgb_out), stream)
        self.library.check(rc, "srl_sim_render_cameras")

    def set_distractors(self, assets_blob):
        """KukaRandButtonGymEnv-v0 only, before the first reset: simulate the distractor bodies (``srl_sim.model.distractor_blob``).
        Observations, rewards and done flags do not change; the bodies' state is ``get_state(F_DISTRACTORS)``."""
        self._dist_blob = np.ascontiguousarray(assets_blob, dtype=np.float64)
        rc = self._lib.srl_sim_set_distractors(self.handle, self._dist_blob.ctypes.data, self._dist_blob.nbytes)
        self.library.check(rc, "srl_sim_set_distractors")

    # -- state access ------------------------------------------------------------------------
    def get_state(self, field):
        dtype, width = _FIELD_SPEC[field]
        out = np.empty((self.num_envs, width), dtype=dtype)
        rc = self._lib.srl_sim_get_state(self.handle, field, out.ctypes.data, out.nbytes)
        self.library.check(rc, "srl_sim_get_state")
        return out

    def set_state(self, field, values):
        dtype, width = _FIELD_SPEC[field]
        arr = np.ascontiguousarray(np.asarray(values, dtype=dtype).reshape(self.num_envs, width))
        rc = self._lib.srl_sim_set_state(self.handle, field, arr.ctypes.data, arr.nbytes)
        self.library.check(rc, "srl_sim_set_state")

    @property
    def launch_count(self):
        return int(self._lib.srl_sim_launch_count(self.handle))

    def last_kernel_ms(self):
        return float(self._lib.srl_sim_last_kernel_ms(self.handle))


_PKG_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# SRL_SIM_CUDA_LIB lets a developer A/B another build of the SAME sm_90a library (e.g. a code-shape variant)
CUDA_LIBRARY_PATH = os.environ.get("SRL_SIM_CUDA_LIB") or os.path.join(_PKG_ROOT, "csrc", "libsrl_sim_b200.so")
_cuda_library = None


def load_cuda_library():
    """Load the sm_90a library; raises (no CPU fallback) when it has not been built."""
    global _cuda_library
    if _cuda_library is None:
        if not os.path.isfile(CUDA_LIBRARY_PATH):
            raise SimError("CUDA extension %s is missing: run `python __graft_entry__.py build` "
                           "(there is no CPU fallback)" % CUDA_LIBRARY_PATH)
        _cuda_library = SimLibrary(CUDA_LIBRARY_PATH)
    return _cuda_library
