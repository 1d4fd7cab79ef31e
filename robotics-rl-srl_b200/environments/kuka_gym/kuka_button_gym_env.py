"""
``KukaButtonGymEnv`` on the H100-native simulator.

Interface mirrored: environments/kuka_gym/kuka_button_gym_env.py:54-463 of the reference (constructor
keywords, spaces, ``reset``/``step``/``getGroundTruth``/``getTargetPos``/``getArmPos``/``getSRLState``, module
constants, ``getGlobals()``).  The PyBullet world, ``Kuka.applyAction`` (environments/kuka_gym/kuka.py:118-187),
``p.stepSimulation()`` and the contact queries behind ``_reward`` run as one sm_90a kernel behind
``include/srl_sim.h``; this class is an N=1 view on it (gym semantics, no auto-reset).  The np_random draws
of the reference (button placement, the 5 random init actions, the per-step action noise) are made HERE, in
the reference's order, and handed to the kernel, so a seeded run consumes the RNG exactly like the reference.
"""
import numpy as np

from environments.srl_env import SRLGymEnv
from srl_sim import _abi, spaces
from srl_sim.backend import default_backend
from srl_sim.model import KUKA_INIT_JOINT_POSITIONS, load_kuka_scene

#  Number of steps before termination
MAX_STEPS = 1000
N_CONTACTS_BEFORE_TERMINATION = 5
# Terminate the episode if the arm is outside the safety sphere during too much time
N_STEPS_OUTSIDE_SAFETY_SPHERE = 5000
RENDER_HEIGHT = 224
RENDER_WIDTH = 224
Z_TABLE = -0.2
N_DISCRETE_ACTIONS = 6
BUTTON_LINK_IDX = 1
BUTTON_GLIDER_IDX = 1  # Button glider joint
DELTA_V = 0.03  # velocity per physics step.
DELTA_V_CONTINUOUS = 0.0035  # velocity per physics step (for continuous actions).
DELTA_THETA = 0.1  # angular velocity per physics step.
RELATIVE_POS = True  # Use relative position for ground truth
NOISE_STD = 0.01  # Add noise to actions, so the env is not fully deterministic
NOISE_STD_CONTINUOUS = 0.0001
NOISE_STD_JOINTS = 0.002
N_RANDOM_ACTIONS_AT_INIT = 5  # Randomize init arm pos: take 5 random actions
BUTTON_DISTANCE_HEIGHT = 0.28  # Extra height added to the buttons position in the distance calculation


def getGlobals():
    """
    :return: (dict)
    """
    return globals()


class _KukaView(object):
    """Stand-in for the reference's ``self._kuka`` object: only the attributes its callers read."""

    def __init__(self):
        self.joint_positions = list(KUKA_INIT_JOINT_POSITIONS)  # never updated in the reference either (:183)
        self.kuka_uid = 0
        self.kuka_gripper_index = 8
        self.kuka_end_effector_index = 6


class KukaButtonGymEnv(SRLGymEnv):
    """
    Gym wrapper for Kuka environment with a push button

    :param urdf_root: (str) unused (the assets ship with the simulator)
    :param renders: (bool) GUI rendering is not available
    :param is_discrete: (bool) Whether to use discrete or continuous actions
    :param multi_view :(bool) image path only
    :param name: (str) name of the folder where recorded data would be stored
    :param max_distance: (float) Max distance between end effector and the button (for negative reward)
    :param action_repeat: (int) Number of timesteps an action is repeated (here it is equivalent to frameskip)
    :param shape_reward: (bool) Set to true, reward = -distance_to_goal
    :param action_joints: (bool) Set actions to apply to the joint space (7 set-points relative to the initial joint
        vector; needs is_discrete=False -- the reference's own reset() fails for the discrete combination)
    :param record_data: (bool) Set to true, record the states / actions / rewards with ``EpisodeSaver`` (frames by name only)
    :param random_target: (bool) Set the button position to a random position on the table
    :param force_down: (bool) Set Down as the only vertical action allowed
    :param state_dim: (int) When learning states
    :param env_rank: (int) the number ID of the environment
    :param srl_pipe: (Queue, [Queue]) contains the input and output of the SRL model
    :param srl_model: (str) The SRL_model used ("ground_truth", "joints", "joints_position")
    :param device: (int) CUDA device ordinal (extension; default 0)
    """
    _ENV_ID = "KukaButtonGymEnv-v0"
    _MAX_STEPS = MAX_STEPS

    def __init__(self, urdf_root=None, renders=False, is_discrete=True, multi_view=False, name="kuka_button_gym",
                 max_distance=0.8, action_repeat=1, shape_reward=False, action_joints=False, record_data=False,
                 random_target=False, force_down=True, state_dim=-1, learn_states=False, verbose=False,
                 save_path='srl_zoo/data/', env_rank=0, srl_pipe=None, srl_model="raw_pixels", device=None, **_):
        super(KukaButtonGymEnv, self).__init__(srl_model=srl_model, relative_pos=RELATIVE_POS, env_rank=env_rank,
                                               srl_pipe=srl_pipe)
        if action_joints and is_discrete:
            # the reference constructs this combination but its reset() dies with an IndexError (a 5-element discrete
            # action reaches Kuka.applyAction's 9-element joint branch, kuka.py:158-161); fail early and clearly instead
            raise ValueError("action_joints requires is_discrete=False")
        self._timestep = 1. / 240.
        self._urdf_root = urdf_root
        self._action_repeat = action_repeat
        self._observation = []
        self._env_step_counter = 0
        self._renders = renders
        self._width = RENDER_WIDTH
        self._height = RENDER_HEIGHT
        self._max_distance = max_distance
        self._shape_reward = shape_reward
        self._random_target = random_target
        self._force_down = force_down
        self._is_discrete = is_discrete
        self.terminated = False
        self.n_contacts = 0
        self.state_dim = state_dim
        self.action_joints = action_joints
        self.relative_pos = RELATIVE_POS
        self.saver = None
        self.multi_view = multi_view
        self.verbose = verbose
        self.max_steps = MAX_STEPS
        self.n_steps_outside = 0
        self.button_pos = None
        self._kuka = _KukaView()
        self.action = None
        self.srl_model = srl_model

        if self._is_discrete:
            self.action_space = spaces.Discrete(N_DISCRETE_ACTIONS)
        else:
            if self.action_joints:
                action_dim = 7  # 7 angles for the arm rotation, from -1 to 1
            else:
                action_dim = 3  # 3 directions for the arm movement, from -1 to 1
            self._action_bound = 1
            action_high = np.array([self._action_bound] * action_dim)
            self.action_space = spaces.Box(-action_high, action_high, dtype=np.float32)

        if self.srl_model == "ground_truth":
            self.state_dim = self.getGroundTruthDim()
        elif self.srl_model == "joints":
            self.state_dim = self.getJointsDim()
        elif self.srl_model == "joints_position":
            self.state_dim = self.getGroundTruthDim() + self.getJointsDim()

        if self.srl_model == "raw_pixels":
            self.observation_space = spaces.Box(low=0, high=255, shape=(self._height, self._width, 6 if multi_view else 3), dtype=np.uint8)
        else:
            self.observation_space = spaces.Box(low=-np.inf, high=np.inf, shape=(self.state_dim,), dtype=np.float32)

        if record_data:   # (:124-126) states, actions, rewards, targets; frames by name only (no rasteriser)
            from state_representation.episode_saver import EpisodeSaver
            self.saver = EpisodeSaver(name, max_distance, state_dim, globals_=getGlobals(), relative_pos=RELATIVE_POS,
                                      learn_states=learn_states, path=save_path)

        if _.get("distractors", False):
            raise ValueError("distractors=True is only available for KukaRandButtonGymEnv-v0 (got %s)" % self._ENV_ID)
        self._backend = default_backend(device)
        self._sim = self._backend.make_sim(self._ENV_ID, 1, seed=0, model_blob=load_kuka_scene().blob,
                                           is_discrete=is_discrete, random_target=random_target, force_down=force_down,
                                           shape_reward=shape_reward, action_repeat=action_repeat,
                                           action_joints=action_joints, max_distance=max_distance, max_steps=self._MAX_STEPS, no_auto_reset=True)
        be = self._backend
        self._obs_buf = be.zeros((1, 3), np.float32)
        self._rew_buf = be.zeros((1,), np.float32)
        self._done_buf = be.zeros((1,), np.uint8)
        self._arm_pos = np.zeros(3)

    # ---- reference surface -------------------------------------------------------------------
    def getSRLState(self, observation):
        state = []
        if self.srl_model in ["ground_truth", "joints_position"]:
            if self.relative_pos:
                state += list(self.getGroundTruth() - self.getTargetPos())
            else:
                state += list(self.getGroundTruth())
        if self.srl_model in ["joints", "joints_position"]:
            state += list(self._kuka.joint_positions)
        if len(state) != 0:
            return np.array(state)
        self.srl_pipe[0].put((self.env_rank, observation))
        return self.srl_pipe[1][self.env_rank].get()

    def getTargetPos(self):
        return self.button_pos

    @staticmethod
    def getJointsDim():
        """
        :return: (int)
        """
        return 14

    @staticmethod
    def getGroundTruthDim():
        return 3

    def getGroundTruth(self):
        return np.array(self.getArmPos())

    def getArmPos(self):
        """
        :return: ([float]) Position (x, y, z) of kuka gripper
        """
        return tuple(self._arm_pos)

    def _pull_state(self):
        self._arm_pos = self._sim.get_state(_abi.F_ROBOT_POS)[0].copy()
        self.button_pos = self._sim.get_state(_abi.F_TARGET_POS)[0].copy()
        c = self._sim.get_state(_abi.F_COUNTERS)[0]
        self.n_contacts, self.n_steps_outside, self.terminated = int(c[0]), int(c[1]), bool(c[2])
        self._env_step_counter = int(self._sim.get_state(_abi.F_STEP_COUNTER)[0, 0])

    def _draw_button_placement(self):
        """np_random draws that place the button (:227-231) -> (x, y) handed to the kernel."""
        x_pos, y_pos = 0.5, 0
        if self._random_target:
            x_pos += 0.15 * self.np_random.uniform(-1, 1)
            y_pos += 0.3 * self.np_random.uniform(-1, 1)
        return [x_pos, y_pos]

    def _reset_draws(self):
        """np_random draws of reset() in the reference's order (:227-231, :250-266) -> the 18 reset values
        (button x, y; 5 x (dx, dy, dz); signed button speed, 0 except for the moving-button variant)."""
        draws = self._draw_button_placement()
        for _ in range(N_RANDOM_ACTIONS_AT_INIT):
            action = [0, 0, 0]
            if self._is_discrete:
                sign = 1 if self.np_random.rand() > 0.5 else -1
                action_idx = self.np_random.randint(3)  # dx, dy or dz
                action[action_idx] += sign * DELTA_V
            elif self.action_joints:
                # joints += DELTA_THETA * np_random.normal(joints.shape): `(7,)` is the MEAN, i.e. one N(7, 1) draw that
                # broadcasts to the seven joints (:257-260); the kernel takes the common set-point offset in the dx slot
                action[0] = float((DELTA_THETA * self.np_random.normal((7,)))[0])
            else:
                rand_direction = self.np_random.normal((3,))
                # L2 normalize, so that the random direction is not too high or too low
                rand_direction /= np.linalg.norm(rand_direction, 2)
                action = list(np.zeros(3) + DELTA_V_CONTINUOUS * rand_direction)
            draws += [float(a) for a in action]
        return draws + [0.0]

    def reset(self):
        draws = self._backend.from_host(np.asarray([self._reset_draws()], dtype=np.float64))
        self._sim.reset(mask=None, reset_draws=draws, obs_out=self._obs_buf, stream=self._backend.stream())
        self._pull_state()
        if self.saver is not None:   # (:275-276)
            self.saver.reset(self._frame_for_saver(), self.getTargetPos(), self.getGroundTruth())
        return self._state_or_image()

    def _frame_for_saver(self):
        """The frame EpisodeSaver stores next to the state (:275-276, :362-363): rendered when images are what the env observes."""
        if self.srl_model == "raw_pixels":
            return self.getExtendedObservation()
        return None

    def _state_or_image(self):
        """What reset() / step() return (:278-281, :365-368): the SRL state, or -- raw_pixels -- the rendered frame."""
        if self.srl_model != "raw_pixels":
            return self.getSRLState(self._observation)
        return np.array(self.getExtendedObservation())

    def getExtendedObservation(self):
        """Image observation of the reference (:287-291): the frame of the fixed camera (two cameras with multi_view)."""
        self._observation = self.render("rgb_array")
        return self._observation

    def step(self, action):
        be = self._backend
        noise = 0.0
        if action is None:
            # the reference steps with a zero action and draws no noise (:295-299)
            # (joints mode: the initial joint vector, i.e. a zero action on the relative set-points)
            act = np.asarray([-1], dtype=np.int32) if self._is_discrete else np.zeros((1, 7 if self.action_joints else 3), dtype=np.float32)
        else:
            self.action = action
            if self._is_discrete:
                noise = self.np_random.normal(0.0, scale=NOISE_STD)
                act = np.asarray([int(action)], dtype=np.int32)
            elif self.action_joints:
                noise = self.np_random.normal(0.0, scale=NOISE_STD_JOINTS)
                act = np.asarray(action, dtype=np.float32).reshape(1, 7)
            else:
                noise = self.np_random.normal(0.0, scale=NOISE_STD_CONTINUOUS)
                act = np.asarray(action, dtype=np.float32).reshape(1, 3)
        self._sim.step(be.from_host(act), noise=be.from_host(np.asarray([noise], dtype=np.float32)),
                       obs_out=self._obs_buf, rew_out=self._rew_buf, done_out=self._done_buf, stream=be.stream())
        rew = float(be.to_host(self._rew_buf)[0])
        done = bool(be.to_host(self._done_buf)[0])
        self._pull_state()
        reward = rew if self._shape_reward else int(rew)
        if self.saver is not None:   # (:362-363)
            self.saver.step(self._frame_for_saver(), self.action, reward, done, self.getGroundTruth())
        return self._state_or_image(), reward, done, {}

    def render(self, mode='human', close=False):
        if mode != "rgb_array":
            return np.array([])
        from srl_sim.render import KUKA_CAMERA, KUKA_CAMERA_2, render_batch
        cams = [KUKA_CAMERA, KUKA_CAMERA_2] if self.multi_view else [KUKA_CAMERA]      # (:385-418)
        return self._backend.to_host(render_batch(self._sim, self._backend, cams, self._width, self._height))[0].copy()

    def close(self):
        if getattr(self, "_sim", None) is not None:
            self._sim.close()
            self._sim = None

    def _termination(self):
        return self.terminated or self._env_step_counter > self.max_steps
