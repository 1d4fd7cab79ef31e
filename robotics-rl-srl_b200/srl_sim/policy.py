"""
ctypes binding of ``include/srl_policy.h``: the per-step helpers of a GPU-resident PPO2 rollout that live in the same
sm_90a library as the simulator -- the policy step (both 64-64 towers, sample, log-probability, value, rollout-buffer writes
in ONE launch) and the VecNormalize observation filter (ONE launch; with ``--num-stack k`` the frame stack step and the filter share it).  With ``srl_sim_step`` a captured rollout is then three
launches per env step instead of ~60 small torch kernels around the simulator's.

Reference pieces replaced: stable-baselines' ``PPO2`` runner ``model.step(obs)`` with ``MlpPolicy`` (selected by
``rl_baselines/rl_algorithm/ppo2.py:58-72``) and ``VecNormalize._obfilt`` (``rl_baselines/utils.py:224-227``).
There is no CPU fallback here either: :class:`FusedPolicy` needs the CUDA library and CUDA tensors.
"""
import ctypes
from ctypes import POINTER, Structure, byref, c_double, c_float, c_int, c_int32, c_int64, c_size_t, c_uint32, c_uint64, c_void_p

HIDDEN, MAX_OBS, MAX_OUT = 64, 32, 8     # observation widths 1..8 and 9..32 (stacked states) run separate kernel instantiations
POLICY_EXPORTS = ["srl_policy_act", "srl_obs_filter", "srl_obs_stack_filter", "srl_ppo2_grad", "srl_ppo2_workspace_bytes", "srl_ppo2_gae",
                  "srl_a2c_grad", "srl_a2c_workspace_bytes", "srl_clip_rmsprop", "srl_dqn_act", "srl_dqn_target", "srl_dqn_grad", "srl_clip_adam",
                  "srl_replay_add", "srl_replay_sample", "srl_replay_update", "srl_sac_arena_floats", "srl_sac_workspace_bytes", "srl_sac_act",
                  "srl_sac_store", "srl_sac_prepare", "srl_sac_grad", "srl_sac_adam"]
GRAD_NAMES = ["pi_w1", "pi_b1", "pi_w2", "pi_b2", "pi_w3", "pi_b3", "vf_w1", "vf_b1", "vf_w2", "vf_b2", "vf_w3", "vf_b3", "logstd"]


class SrlMlpPolicy(Structure):
    """struct srl_mlp_policy (include/srl_policy.h)."""
    _fields_ = [("struct_size", c_uint32), ("obs_dim", c_int32), ("n_out", c_int32), ("discrete", c_int32)] + \
               [(name, c_void_p) for name in ("pi_w1", "pi_b1", "pi_w2", "pi_b2", "pi_w3", "pi_b3",
                                              "vf_w1", "vf_b1", "vf_w2", "vf_b2", "vf_w3", "vf_b3", "logstd")]


class SrlMlpGrads(Structure):
    """struct srl_mlp_grads (include/srl_policy.h)."""
    _fields_ = [("struct_size", c_uint32), ("reserved", c_uint32)] + \
               [(name, c_void_p) for name in ("pi_w1", "pi_b1", "pi_w2", "pi_b2", "pi_w3", "pi_b3",
                                              "vf_w1", "vf_b1", "vf_w2", "vf_b2", "vf_w3", "vf_b3", "logstd")]


class SrlReplayTree(Structure):
    """struct srl_replay_tree (include/srl_policy.h)."""
    _fields_ = [("struct_size", c_uint32), ("n_envs", c_int32), ("capacity", c_int64), ("tree_cap", c_int64)] + \
               [(name, c_void_p) for name in ("sum", "min", "max_priority", "size", "stamp")]


class SrlSacNets(Structure):
    """struct srl_sac_nets (include/srl_policy.h)."""
    _fields_ = [("struct_size", c_uint32), ("obs_dim", c_int32), ("act_dim", c_int32), ("reserved", c_int32), ("arena", c_void_p), ("target", c_void_p)]


def bind(cdll):
    """Declare the argument types of the two entry points on a loaded library (raises AttributeError if they are missing)."""
    cdll.srl_policy_act.restype = c_int
    cdll.srl_policy_act.argtypes = [POINTER(SrlMlpPolicy), c_int, c_void_p, c_void_p, c_uint64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]
    cdll.srl_obs_filter.restype = c_int
    cdll.srl_obs_filter.argtypes = [c_int, c_int, c_void_p, c_void_p, c_int, c_float, c_float, c_void_p, c_void_p]
    cdll.srl_obs_stack_filter.restype = c_int
    cdll.srl_obs_stack_filter.argtypes = [c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_float, c_float, c_void_p, c_void_p]
    cdll.srl_ppo2_workspace_bytes.restype = c_size_t
    cdll.srl_ppo2_workspace_bytes.argtypes = [c_int, c_int, c_int, c_int]
    cdll.srl_ppo2_grad.restype = c_int
    cdll.srl_ppo2_grad.argtypes = [POINTER(SrlMlpPolicy), POINTER(SrlMlpGrads), c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                   c_float, c_float, c_float, c_void_p, c_size_t, c_void_p]
    cdll.srl_ppo2_gae.restype = c_int
    cdll.srl_ppo2_gae.argtypes = [c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_double, c_double, c_void_p, c_void_p, c_void_p]
    cdll.srl_a2c_workspace_bytes.restype = c_size_t
    cdll.srl_a2c_workspace_bytes.argtypes = [c_int, c_int, c_int, c_int]
    cdll.srl_a2c_grad.restype = c_int
    cdll.srl_a2c_grad.argtypes = [POINTER(SrlMlpPolicy), POINTER(SrlMlpGrads), c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_float,
                                  c_void_p, c_size_t, c_void_p]
    cdll.srl_clip_rmsprop.restype = c_int
    cdll.srl_clip_rmsprop.argtypes = [c_int, c_int, c_int, POINTER(SrlMlpGrads), POINTER(SrlMlpGrads), POINTER(SrlMlpGrads), c_void_p, c_float, c_float,
                                      c_float, c_void_p]
    P, G = POINTER(SrlMlpPolicy), POINTER(SrlMlpGrads)
    cdll.srl_dqn_act.restype = c_int
    cdll.srl_dqn_act.argtypes = [P, c_int, c_void_p, c_void_p, c_void_p, c_uint64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]
    cdll.srl_dqn_target.restype = c_int
    cdll.srl_dqn_target.argtypes = [P, P, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_void_p, c_void_p]
    cdll.srl_dqn_grad.restype = c_int
    cdll.srl_dqn_grad.argtypes = [P, G, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]
    cdll.srl_clip_adam.restype = c_int
    cdll.srl_clip_adam.argtypes = [c_int, c_int, c_int, G, G, G, G, c_void_p, c_void_p, c_float, c_float, c_float, c_float, c_void_p]
    T = POINTER(SrlReplayTree)
    cdll.srl_replay_add.restype = c_int
    cdll.srl_replay_add.argtypes = [T, c_int64, c_double, c_void_p]
    cdll.srl_replay_sample.restype = c_int
    cdll.srl_replay_sample.argtypes = [T, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]
    cdll.srl_replay_update.restype = c_int
    cdll.srl_replay_update.argtypes = [T, c_int, c_void_p, c_void_p, c_double, c_float, c_void_p]
    S = POINTER(SrlSacNets)
    cdll.srl_sac_arena_floats.restype = c_size_t
    cdll.srl_sac_arena_floats.argtypes = [c_int, c_int]
    cdll.srl_sac_workspace_bytes.restype = c_size_t
    cdll.srl_sac_workspace_bytes.argtypes = [c_int, c_int, c_int]
    cdll.srl_sac_act.restype = c_int
    cdll.srl_sac_act.argtypes = [S, c_int, c_void_p, c_int, c_void_p, c_uint64, c_void_p, c_void_p]
    cdll.srl_sac_store.restype = c_int
    cdll.srl_sac_store.argtypes = [c_int, c_int, c_int, c_int] + [c_void_p] * 12
    cdll.srl_sac_prepare.restype = c_int
    cdll.srl_sac_prepare.argtypes = [S, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_float, c_int, c_float, c_float,
                                     c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]
    cdll.srl_sac_grad.restype = c_int
    cdll.srl_sac_grad.argtypes = [S, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]
    cdll.srl_sac_adam.restype = c_int
    cdll.srl_sac_adam.argtypes = [S, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_float, c_float, c_int, c_float, c_void_p]
    return cdll


def policy_params(policy):
    """The parameters of an MlpPolicy in the order of ``srl_mlp_grads`` (logstd last, Box only)."""
    lin = lambda tower: [m for m in tower if hasattr(m, "weight")]
    params = [t for layer in lin(policy.pi) + lin(policy.vf) for t in (layer.weight, layer.bias)]
    return params if policy.discrete else params + [policy.logstd]


def tensors_struct(tensors):
    """``srl_mlp_grads`` over 12 or 13 tensors in the order of :func:`policy_params` (gradients, parameters or optimiser slots)."""
    s = SrlMlpGrads()
    s.struct_size = ctypes.sizeof(SrlMlpGrads)
    for name, t in zip(GRAD_NAMES, tensors):
        setattr(s, name, t.data_ptr())
    return s


def policy_struct(policy):
    """``srl_mlp_policy`` over the parameters of an ``rl_baselines.ppo2.MlpPolicy`` (pointers into the live tensors: optimiser
    steps are seen by the next launch).  Returns (struct, keep-alive list)."""
    lin = lambda tower: [m for m in tower if hasattr(m, "weight")]
    pi, vf = lin(policy.pi), lin(policy.vf)
    tensors = []
    for layer in pi + vf:
        for t in (layer.weight, layer.bias):
            if not t.is_contiguous() or str(t.dtype) != "torch.float32":
                raise ValueError("policy parameters must be contiguous float32")
            tensors.append(t)
    obs_dim, n_out = pi[0].weight.shape[1], pi[2].weight.shape[0]
    if pi[0].weight.shape[0] != HIDDEN or pi[1].weight.shape != (HIDDEN, HIDDEN) or vf[2].weight.shape[0] != 1:
        raise ValueError("srl_policy_act implements the 64-64 MlpPolicy")
    if not (1 <= obs_dim <= MAX_OBS and 1 <= n_out <= MAX_OUT):
        raise ValueError("unsupported policy shape obs_dim=%d n_out=%d" % (obs_dim, n_out))
    s = SrlMlpPolicy()
    s.struct_size = ctypes.sizeof(SrlMlpPolicy)
    s.obs_dim, s.n_out, s.discrete = obs_dim, n_out, int(policy.discrete)
    for name, t in zip(("pi_w1", "pi_b1", "pi_w2", "pi_b2", "pi_w3", "pi_b3", "vf_w1", "vf_b1", "vf_w2", "vf_b2", "vf_w3", "vf_b3"), tensors):
        setattr(s, name, t.data_ptr())
    s.logstd = None if policy.discrete else policy.logstd.data_ptr()
    return s, tensors


class FusedPolicy(object):
    """The fused policy step + observation filter on the CUDA library, for one ``MlpPolicy`` and one env batch."""

    def __init__(self, library, policy, filter_state, seed, env_offset=0, clip=10.0, eps=1e-8):
        """
        :param library: (srl_sim._abi.SimLibrary) the loaded CUDA library
        :param policy: (rl_baselines.ppo2.MlpPolicy) on a CUDA device
        :param filter_state: (torch.Tensor) float64 [2 * obs_dim + 1] on the same device: mean, var, count (updated in place)
        :param seed: (int) key of the sampling streams; env ``i`` uses the stream (seed, env_offset + i)
        """
        import torch
        self._lib = bind(library.lib)
        self._library = library
        self.struct, self._keep = policy_struct(policy)
        dev = policy.pi[0].weight.device
        if dev.type != "cuda":
            raise ValueError("FusedPolicy needs a policy on a CUDA device (there is no CPU fallback)")
        if filter_state.dtype != torch.float64 or filter_state.numel() != 2 * self.struct.obs_dim + 1 or not filter_state.is_contiguous():
            raise ValueError("filter_state must be a contiguous float64 tensor of 2 * obs_dim + 1 elements")
        self.filter_state = filter_state
        self.rng = torch.tensor([int(seed) & 0x7FFFFFFFFFFFFFFF, 0, 0], dtype=torch.int64, device=dev)   # {seed, step counter, arrivals}
        self.env_offset, self.clip, self.eps = int(env_offset), float(clip), float(eps)
        self.obs_dim, self.n_out, self.discrete = self.struct.obs_dim, self.struct.n_out, bool(self.struct.discrete)

    def act(self, n, obs, act_env, logp, value, obs_buf=None, act_buf=None, stream=None):
        rc = self._lib.srl_policy_act(byref(self.struct), int(n), obs.data_ptr(), self.rng.data_ptr(), self.env_offset,
                                      None if obs_buf is None else obs_buf.data_ptr(), act_env.data_ptr(),
                                      None if act_buf is None else act_buf.data_ptr(), logp.data_ptr(), value.data_ptr(), stream)
        self._library.check(rc, "srl_policy_act")

    def filter(self, n, obs_raw, obs_norm_out, update=True, stream=None):
        rc = self._lib.srl_obs_filter(int(n), self.obs_dim, obs_raw.data_ptr(), self.filter_state.data_ptr(), int(bool(update)),
                                      self.clip, self.eps, obs_norm_out.data_ptr(), stream)
        self._library.check(rc, "srl_obs_filter")

    def stack_filter(self, n, obs_raw, done, stack, obs_norm_out, update=True, stream=None):
        """``srl_obs_stack_filter``: VecFrameStack + VecNormalize in one launch.  ``obs_raw`` float32 [n, D] with ``obs_dim`` a multiple k of D,
        ``done`` uint8 [n] (None: a reset, every row starts from zeros), ``stack`` float32 [n, k D] advanced in place, ``obs_norm_out``
        float32 [n, k D]; the filter state is this object's (2 k D + 1 doubles)."""
        D = int(obs_raw.shape[-1])
        if D < 1 or self.obs_dim % D:
            raise ValueError("stack_filter: the policy width %d is not a multiple of the observation width %d" % (self.obs_dim, D))
        rc = self._lib.srl_obs_stack_filter(int(n), D, self.obs_dim // D, obs_raw.data_ptr(), None if done is None else done.data_ptr(), stack.data_ptr(),
                                            self.filter_state.data_ptr(), int(bool(update)), self.clip, self.eps, obs_norm_out.data_ptr(), stream)
        self._library.check(rc, "srl_obs_stack_filter")


class FusedPPO2Grad(object):
    """``srl_ppo2_grad``: the gradient of the PPO2 loss over one minibatch in one pass (forward, loss derivative, backward of both towers
    with every activation on chip), written into the policy's ``.grad`` tensors -- what ``loss.backward()`` of
    ``rl_baselines.ppo2``'s minibatch step produces.  Gradient clipping and the optimiser step stay with torch."""
    _workspace_fn = "srl_ppo2_workspace_bytes"

    def __init__(self, library, policy, minibatch):
        import torch
        self._lib = bind(library.lib)
        self._library = library
        self.struct, self._keep = policy_struct(policy)
        dev = policy.pi[0].weight.device
        if dev.type != "cuda":
            raise ValueError("FusedPPO2Grad needs a policy on a CUDA device (there is no CPU fallback)")
        params = policy_params(policy)
        for prm in params:
            prm.grad = torch.zeros_like(prm)               # static gradient tensors: the kernel overwrites them, the optimiser reads them (capturable)
        self.grads = tensors_struct([prm.grad for prm in params])
        self.params = params
        self.minibatch = int(minibatch)
        nbytes = int(getattr(self._lib, self._workspace_fn)(self.struct.obs_dim, self.struct.n_out, self.struct.discrete, self.minibatch))
        if nbytes <= 0:
            raise ValueError("%s: unsupported shape" % self._workspace_fn)
        self.workspace = torch.zeros(nbytes, dtype=torch.uint8, device=dev)

    def gae(self, rew, value, done, last_value, gamma, lam, adv_out, ret_out, stream=None):
        """``srl_ppo2_gae``: GAE(lambda) of a [T, N] rollout in one launch (float32 tensors; ``done`` holds 1.0 where an episode ended)."""
        T, N = rew.shape
        rc = self._lib.srl_ppo2_gae(int(T), int(N), rew.data_ptr(), value.data_ptr(), done.data_ptr(), last_value.data_ptr(), float(gamma), float(lam),
                                    adv_out.data_ptr(), ret_out.data_ptr(), stream)
        self._library.check(rc, "srl_ppo2_gae")

    def __call__(self, idx, obs, actions, adv, ret, old_logp, old_value, cliprange, ent_coef, vf_coef, stream=None):
        """All arguments are CUDA tensors of the whole rollout (``idx``: int64 [minibatch] rows, or None for the first ``minibatch`` rows)."""
        rc = self._lib.srl_ppo2_grad(byref(self.struct), byref(self.grads), self.minibatch, None if idx is None else idx.data_ptr(), obs.data_ptr(),
                                     actions.data_ptr(), adv.data_ptr(), ret.data_ptr(), old_logp.data_ptr(), old_value.data_ptr(),
                                     float(cliprange), float(ent_coef), float(vf_coef), self.workspace.data_ptr(), self.workspace.numel(), stream)
        self._library.check(rc, "srl_ppo2_grad")


class FusedA2CGrad(FusedPPO2Grad):
    """``srl_a2c_grad``: the gradient of stable-baselines' A2C loss over the rows of one update (advantage ``ret - old_value``, no
    normalisation, no clipping; include/srl_policy.h), in the same kernels as :class:`FusedPPO2Grad` and into the same static ``.grad``
    tensors.  ``minibatch`` is the number of rows of an update (n_steps x envs).  ``gae`` (lambda = 1) gives the returns."""
    _workspace_fn = "srl_a2c_workspace_bytes"

    def __call__(self, idx, obs, actions, ret, old_value, ent_coef, vf_coef, stream=None):
        """CUDA tensors of the rollout (``idx``: int64 [rows], or None for the first ``minibatch`` rows)."""
        rc = self._lib.srl_a2c_grad(byref(self.struct), byref(self.grads), self.minibatch, None if idx is None else idx.data_ptr(), obs.data_ptr(),
                                    actions.data_ptr(), ret.data_ptr(), old_value.data_ptr(), float(ent_coef), float(vf_coef),
                                    self.workspace.data_ptr(), self.workspace.numel(), stream)
        self._library.check(rc, "srl_a2c_grad")


class FusedClipRMSprop(object):
    """``srl_clip_rmsprop``: TF1's ``clip_by_global_norm`` + ``RMSPropOptimizer`` (momentum 0) over every tensor of an MlpPolicy in one launch.
    Reads the policy's ``.grad`` tensors (which must exist and stay put: :class:`FusedA2CGrad` makes them static), updates the parameters in
    place and owns the RMSProp slots ``ms`` (initialised to 1.0 as TF does) and the learning rate ``lr`` (float32 [1] on the device, for
    a captured step to follow a schedule)."""

    def __init__(self, library, policy, max_grad_norm, alpha, epsilon, lr=None):
        import torch
        self._lib = bind(library.lib)
        self._library = library
        self.params = policy_params(policy)
        dev = self.params[0].device
        if dev.type != "cuda":
            raise ValueError("FusedClipRMSprop needs a policy on a CUDA device (there is no CPU fallback)")
        if any(p.grad is None for p in self.params):
            raise ValueError("FusedClipRMSprop needs the policy's .grad tensors (create them first, e.g. with FusedA2CGrad)")
        st, _ = policy_struct(policy)
        self.obs_dim, self.n_out, self.discrete = st.obs_dim, st.n_out, st.discrete
        self.ms = [torch.ones_like(p) for p in self.params]
        self.lr = torch.zeros(1, dtype=torch.float32, device=dev) if lr is None else lr
        self._p, self._g, self._m = tensors_struct(self.params), tensors_struct([p.grad for p in self.params]), tensors_struct(self.ms)
        self.max_grad_norm, self.alpha, self.epsilon = float(max_grad_norm), float(alpha), float(epsilon)

    def __call__(self, lr=None, stream=None):
        """One step with the learning rate in ``lr`` (a float32 device scalar; default: this object's ``lr``)."""
        lr = self.lr if lr is None else lr
        rc = self._lib.srl_clip_rmsprop(self.obs_dim, self.n_out, self.discrete, byref(self._p), byref(self._g), byref(self._m), lr.data_ptr(),
                                        self.max_grad_norm, self.alpha, self.epsilon, stream)
        self._library.check(rc, "srl_clip_rmsprop")


# ---- DQN (include/srl_policy.h: srl_dqn_*, srl_replay_*, srl_clip_adam; rl_baselines/deepq.py) ----

def _cuda_policy_struct(lib_name, policy):
    st, keep = policy_struct(policy)
    if policy.pi[0].weight.device.type != "cuda":
        raise ValueError("%s needs a network on a CUDA device (there is no CPU fallback)" % lib_name)
    if not st.discrete:
        raise ValueError("%s: the Q network must be discrete" % lib_name)
    return st, keep


class FusedDQNAct(object):
    """``srl_dqn_act``: the epsilon-greedy step of a dueling Q network (``rl_baselines.deepq.DuelingQ``) for one env batch, in one launch.
    Owns the sampling record ``rng`` {seed, counter, 0} and the exploration rate ``eps`` (float32 [1] on the device)."""

    def __init__(self, library, qnet, seed, env_offset=0):
        import torch
        self._lib = bind(library.lib)
        self._library = library
        self.struct, self._keep = _cuda_policy_struct("FusedDQNAct", qnet)
        dev = qnet.pi[0].weight.device
        self.rng = torch.tensor([int(seed) & 0x7FFFFFFFFFFFFFFF, 0, 0], dtype=torch.int64, device=dev)
        self.eps = torch.zeros(1, dtype=torch.float32, device=dev)
        self.env_offset = int(env_offset)

    def __call__(self, n, obs, act_env, obs_buf=None, act_buf=None, q_out=None, eps=None, stream=None):
        """``eps``: a float32 device scalar to read the exploration rate from (default: this object's ``eps``)."""
        ptr = lambda t: None if t is None else t.data_ptr()
        rc = self._lib.srl_dqn_act(byref(self.struct), int(n), obs.data_ptr(), (self.eps if eps is None else eps).data_ptr(), self.rng.data_ptr(), self.env_offset, ptr(obs_buf),
                                   act_env.data_ptr(), ptr(act_buf), ptr(q_out), stream)
        self._library.check(rc, "srl_dqn_act")


class FusedDQNTarget(object):
    """``srl_dqn_target``: the double-Q targets ``y`` of a sampled batch from the online and the target network (both live tensors)."""

    def __init__(self, library, online, target):
        self._lib = bind(library.lib)
        self._library = library
        self.online, self._keep_o = _cuda_policy_struct("FusedDQNTarget", online)
        self.target, self._keep_t = _cuda_policy_struct("FusedDQNTarget", target)

    def __call__(self, batch, idx, next_obs, rew, done, gamma, y, stream=None):
        rc = self._lib.srl_dqn_target(byref(self.online), byref(self.target), int(batch), None if idx is None else idx.data_ptr(), next_obs.data_ptr(),
                                      rew.data_ptr(), done.data_ptr(), float(gamma), y.data_ptr(), stream)
        self._library.check(rc, "srl_dqn_target")


class FusedDQNGrad(FusedPPO2Grad):
    """``srl_dqn_grad``: the gradient of ``mean(w huber(Q(s, a) - y))`` over a batch of ``minibatch`` samples, in the kernels of
    :class:`FusedPPO2Grad`, into the network's static ``.grad`` tensors; also writes the per-sample td."""
    _workspace_fn = "srl_a2c_workspace_bytes"

    def __call__(self, idx, obs, actions, y, weights, td_out, stream=None):
        rc = self._lib.srl_dqn_grad(byref(self.struct), byref(self.grads), self.minibatch, None if idx is None else idx.data_ptr(), obs.data_ptr(),
                                    actions.data_ptr(), y.data_ptr(), None if weights is None else weights.data_ptr(), td_out.data_ptr(),
                                    self.workspace.data_ptr(), self.workspace.numel(), stream)
        self._library.check(rc, "srl_dqn_grad")


class FusedClipAdam(object):
    """``srl_clip_adam``: ``tf.clip_by_norm`` per tensor + one TF1 Adam step over every tensor of the network in one launch.  Reads the
    ``.grad`` tensors (static: :class:`FusedDQNGrad` makes them), owns the slots ``m``, ``v`` (zeros), TF's ``beta_power`` accumulators
    {beta1^t, beta2^t} (float32 [2], from {beta1, beta2}) and the learning rate ``lr`` (float32 [1])."""

    def __init__(self, library, policy, clip_norm, beta1=0.9, beta2=0.999, epsilon=1e-8):
        import torch
        self._lib = bind(library.lib)
        self._library = library
        self.params = policy_params(policy)
        dev = self.params[0].device
        if dev.type != "cuda":
            raise ValueError("FusedClipAdam needs a network on a CUDA device (there is no CPU fallback)")
        if any(p.grad is None for p in self.params):
            raise ValueError("FusedClipAdam needs the network's .grad tensors (create them first, e.g. with FusedDQNGrad)")
        st, _ = policy_struct(policy)
        self.obs_dim, self.n_out, self.discrete = st.obs_dim, st.n_out, st.discrete
        self.m = [torch.zeros_like(p) for p in self.params]
        self.v = [torch.zeros_like(p) for p in self.params]
        self.beta_power = torch.tensor([beta1, beta2], dtype=torch.float32, device=dev)
        self.lr = torch.zeros(1, dtype=torch.float32, device=dev)
        self._p, self._g = tensors_struct(self.params), tensors_struct([p.grad for p in self.params])
        self._m, self._v = tensors_struct(self.m), tensors_struct(self.v)
        self.clip_norm, self.beta1, self.beta2, self.epsilon = float(clip_norm), float(beta1), float(beta2), float(epsilon)

    def __call__(self, stream=None):
        rc = self._lib.srl_clip_adam(self.obs_dim, self.n_out, self.discrete, byref(self._p), byref(self._g), byref(self._m), byref(self._v),
                                     self.lr.data_ptr(), self.beta_power.data_ptr(), self.clip_norm, self.beta1, self.beta2, self.epsilon, stream)
        self._library.check(rc, "srl_clip_adam")


class FusedReplay(object):
    """baselines' prioritized replay over a ring of ``rows`` x ``n_envs`` transitions on the device (``srl_replay_*``): the two float64
    segment trees, ``max_priority``, the stored count ``size``, the sampling record ``rng`` and the importance exponent ``beta`` (float64 [1]).
    ``sum`` / ``min`` are [2 tree_cap] with the root at 1 and leaf i at tree_cap + i."""

    def __init__(self, library, rows, n_envs, seed, alpha, device):
        import torch
        self._lib = bind(library.lib)
        self._library = library
        capacity = int(rows) * int(n_envs)
        tree_cap = 1
        while tree_cap < capacity:
            tree_cap *= 2
        self.alpha, self.n_envs, self.capacity, self.tree_cap = float(alpha), int(n_envs), capacity, tree_cap
        self.sum = torch.zeros(2 * tree_cap, dtype=torch.float64, device=device)
        self.min = torch.full((2 * tree_cap,), float("inf"), dtype=torch.float64, device=device)
        self.max_priority = torch.ones(1, dtype=torch.float64, device=device)
        self.size = torch.zeros(1, dtype=torch.int64, device=device)
        self.stamp = torch.full((capacity,), -1, dtype=torch.int32, device=device)
        self.rng = torch.tensor([int(seed) & 0x7FFFFFFFFFFFFFFF, 0, 0], dtype=torch.int64, device=device)
        self.beta = torch.zeros(1, dtype=torch.float64, device=device)
        t = SrlReplayTree()
        t.struct_size = ctypes.sizeof(SrlReplayTree)
        t.n_envs, t.capacity, t.tree_cap = self.n_envs, capacity, tree_cap
        for name in ("sum", "min", "max_priority", "size", "stamp"):
            setattr(t, name, getattr(self, name).data_ptr())
        self.struct = t

    def add(self, row, stream=None):
        self._library.check(self._lib.srl_replay_add(byref(self.struct), int(row), self.alpha, stream), "srl_replay_add")

    def sample(self, batch, idx_out, w_out, prioritized=True, beta=None, stream=None):
        """``beta``: a float64 device scalar to read the importance exponent from (default: this object's ``beta``)."""
        rc = self._lib.srl_replay_sample(byref(self.struct), int(batch), int(bool(prioritized)), (self.beta if beta is None else beta).data_ptr(), self.rng.data_ptr(),
                                         idx_out.data_ptr(), w_out.data_ptr(), stream)
        self._library.check(rc, "srl_replay_sample")

    def update(self, batch, idx, td, eps, stream=None):
        rc = self._lib.srl_replay_update(byref(self.struct), int(batch), idx.data_ptr(), td.data_ptr(), self.alpha, float(eps), stream)
        self._library.check(rc, "srl_replay_update")


# ---- SAC (include/srl_policy.h: srl_sac_*; rl_baselines/sac.py) ----

class _FusedSAC(object):
    """The library and the ``srl_sac_nets`` of an ``rl_baselines.sac.SACNets`` (its parameter arena and target, live on a CUDA device)."""

    def __init__(self, library, nets):
        self._lib = bind(library.lib)
        self._library = library
        if nets.arena.device.type != "cuda":
            raise ValueError("%s needs the networks on a CUDA device (there is no CPU fallback)" % type(self).__name__)
        if int(self._lib.srl_sac_arena_floats(nets.obs_dim, nets.act_dim)) != nets.arena.numel():
            raise ValueError("%s: the arena of %d floats is not the layout of srl_sac_arena_floats(%d, %d)" % (type(self).__name__, nets.arena.numel(), nets.obs_dim, nets.act_dim))
        s = SrlSacNets()
        s.struct_size = ctypes.sizeof(SrlSacNets)
        s.obs_dim, s.act_dim, s.arena, s.target = nets.obs_dim, nets.act_dim, nets.arena.data_ptr(), nets.target.data_ptr()
        self.struct, self.nets, self.dev = s, nets, nets.arena.device

    def _check(self, rc, name):
        self._library.check(rc, name)


class FusedSACAct(_FusedSAC):
    """``srl_sac_act``: the action of an env batch, ``mode`` 0 sample, 1 ``tanh(mu)``, 2 uniform random; owns the sampling record ``rng``."""
    SAMPLE, DETERMINISTIC, RANDOM = 0, 1, 2

    def __init__(self, library, nets, seed, env_offset=0):
        import torch
        super().__init__(library, nets)
        self.rng = torch.tensor([int(seed) & 0x7FFFFFFFFFFFFFFF, 0, 0], dtype=torch.int64, device=self.dev)
        self.env_offset = int(env_offset)

    def __call__(self, n, obs, act_out, mode=0, stream=None):
        rc = self._lib.srl_sac_act(byref(self.struct), int(n), None if obs is None else obs.data_ptr(), int(mode), self.rng.data_ptr(), self.env_offset,
                                   act_out.data_ptr(), stream)
        self._check(rc, "srl_sac_act")


class FusedSACStore(object):
    """``srl_sac_store``: one lockstep step into ring row ``step % rows`` (the row read on the device), then ``obs <- new_obs`` and
    ``step += 1``.  Owns ``step`` (int64 [2] {steps stored, 0})."""

    def __init__(self, library, ring, device):
        import torch
        self._lib = bind(library.lib)
        self._library = library
        self.ring = ring
        self.rows, self.n, self.obs_dim = ring["obs"].shape
        self.act_dim = ring["act"].shape[2]
        self.step = torch.zeros(2, dtype=torch.int64, device=device)

    def __call__(self, obs, act, rew, done, new_obs, stream=None):
        r = self.ring
        rc = self._lib.srl_sac_store(self.rows, self.n, self.obs_dim, self.act_dim, self.step.data_ptr(), obs.data_ptr(), act.data_ptr(), rew.data_ptr(),
                                     done.data_ptr(), new_obs.data_ptr(), r["obs"].data_ptr(), r["act"].data_ptr(), r["rew"].data_ptr(), r["done"].data_ptr(),
                                     r["next_obs"].data_ptr(), stream)
        self._library.check(rc, "srl_sac_store")


class FusedSACPrepare(_FusedSAC):
    """``srl_sac_prepare``: sample indices, q_backup, v_backup, logp and the actor's head derivatives of ``batch`` samples; the gradient of
    log_ent_coef goes to ``ent_grad`` (default: its entry of the gradient arena ``grad``).  Owns the sampling record ``rng`` and the outputs."""

    def __init__(self, library, nets, ring, batch, seed, grad, workspace):
        import torch
        super().__init__(library, nets)
        self.ring, self.batch = ring, int(batch)
        self.rows, self.n = ring["obs"].shape[:2]
        z = lambda *shape, dtype=torch.float32: torch.zeros(shape, dtype=dtype, device=self.dev)
        self.rng = torch.tensor([int(seed) & 0x7FFFFFFFFFFFFFFF, 0, 0], dtype=torch.int64, device=self.dev)
        self.idx, self.q_backup, self.v_backup, self.logp = z(batch, dtype=torch.int64), z(batch), z(batch), z(batch)
        self.d_actor = z(batch, 2 * nets.act_dim)
        self.ent_grad, self.workspace = grad[-1:], workspace

    def __call__(self, step, gamma, ent_coef, target_entropy, stream=None):
        """``ent_coef``: a float (fixed) or None ('auto': alpha = exp(log_ent_coef), read on the device)."""
        r = self.ring
        rc = self._lib.srl_sac_prepare(byref(self.struct), self.rows, self.n, step.data_ptr(), r["obs"].data_ptr(), r["act"].data_ptr(), r["rew"].data_ptr(),
                                       r["done"].data_ptr(), r["next_obs"].data_ptr(), self.batch, float(gamma), int(ent_coef is None),
                                       0.0 if ent_coef is None else float(ent_coef), float(target_entropy), self.rng.data_ptr(), self.idx.data_ptr(),
                                       self.q_backup.data_ptr(), self.v_backup.data_ptr(), self.logp.data_ptr(), self.d_actor.data_ptr(),
                                       self.ent_grad.data_ptr(), self.workspace.data_ptr(), self.workspace.numel(), stream)
        self._check(rc, "srl_sac_prepare")


class FusedSACGrad(_FusedSAC):
    """``srl_sac_grad``: the weight gradients of the actor, qf1, qf2 and vf into the gradient arena ``grad`` (every entry but log_ent_coef's)
    from what :class:`FusedSACPrepare` left.  ``workspace(...)`` sizes the scratch both share."""

    @staticmethod
    def workspace(library, nets, batch):
        import torch
        nbytes = int(bind(library.lib).srl_sac_workspace_bytes(nets.obs_dim, nets.act_dim, int(batch)))
        if nbytes <= 0:
            raise ValueError("srl_sac_workspace_bytes: unsupported shape")
        return torch.zeros(nbytes, dtype=torch.uint8, device=nets.arena.device)

    def __call__(self, prep, grad, stream=None):
        r = prep.ring
        rc = self._lib.srl_sac_grad(byref(self.struct), prep.n, r["obs"].data_ptr(), r["act"].data_ptr(), prep.batch, prep.idx.data_ptr(),
                                    prep.q_backup.data_ptr(), prep.v_backup.data_ptr(), prep.d_actor.data_ptr(), grad.data_ptr(), prep.workspace.data_ptr(),
                                    prep.workspace.numel(), stream)
        self._check(rc, "srl_sac_grad")


class FusedSACAdam(_FusedSAC):
    """``srl_sac_adam``: TF1 Adam over the whole arena and the Polyak update of the target in one launch.  Owns the slots ``m``, ``v``,
    TF's ``beta_power`` {beta1^t, beta2^t} (from {beta1, beta2}) and the learning rate ``lr`` (float32 [1])."""

    def __init__(self, library, nets, beta1=0.9, beta2=0.999, epsilon=1e-8, tau=0.005):
        import torch
        super().__init__(library, nets)
        self.m, self.v = torch.zeros_like(nets.arena), torch.zeros_like(nets.arena)
        self.beta_power = torch.tensor([beta1, beta2], dtype=torch.float32, device=self.dev)
        self.lr = torch.zeros(1, dtype=torch.float32, device=self.dev)
        self.beta1, self.beta2, self.epsilon, self.tau = float(beta1), float(beta2), float(epsilon), float(tau)

    def __call__(self, grad, polyak=True, stream=None):
        rc = self._lib.srl_sac_adam(byref(self.struct), grad.data_ptr(), self.m.data_ptr(), self.v.data_ptr(), self.lr.data_ptr(), self.beta_power.data_ptr(),
                                    self.beta1, self.beta2, self.epsilon, int(bool(polyak)), self.tau, stream)
        self._check(rc, "srl_sac_adam")
