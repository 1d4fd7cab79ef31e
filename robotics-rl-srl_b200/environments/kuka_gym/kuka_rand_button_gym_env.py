"""
Mirror of environments/kuka_gym/kuka_rand_button_gym_env.py: the button-push env "with a push button in a
random position and some random objects".  The reference places up to 10 distractor bodies and a sphere that is
kicked at env step 10 (:58-68,117-127).  They are simulated with ``distractors=True`` (opt-in, default off): the
placements use the env's own ``np_random`` draws like the reference, the object types the global ``np.random``
like the reference, and the kick direction the library's counter-based stream (the reference's global, unseeded
draw is not reproducible anyway).  The bodies never push the arm back, so observations, rewards and done flags are
the same with and without them; they show in ``getDistractors()`` and in every rendered frame (``srl_model="raw_pixels"``
observations, ``render()``, ``multi_view`` and the frames ``record_data=True`` saves), the duck, the brick and the cube as the
boxes the asset blob declares, the sphere as a ball (``srl_sim.model.distractor_blob``).
Everything else -- MAX_STEPS, the env RNG draws of reset() -- is identical to KukaButtonGymEnv.
"""
from .kuka_button_gym_env import *  # noqa: F401,F403
from .kuka_button_gym_env import KukaButtonGymEnv
import numpy as np
from srl_sim import _abi

MAX_STEPS = 1000
BALL_FORCE = 10


class KukaRandButtonGymEnv(KukaButtonGymEnv):
    """
    Kuka environment with a push button in a random position (and, with ``distractors=True``, the random objects).
    """
    _ENV_ID = "KukaRandButtonGymEnv-v0"

    def __init__(self, name="kuka_rand_button_gym", distractors=False, **kwargs):
        super(KukaRandButtonGymEnv, self).__init__(name=name, **kwargs)
        self.max_steps = MAX_STEPS
        self.distractors = bool(distractors)
        if self.distractors:
            from srl_sim.model import distractor_blob
            self._sim.set_distractors(distractor_blob())

    def getDistractors(self):
        """The 11 bodies, f64[11, 9]: position, quaternion (x, y, z, w), type (0 duck, 1 lego, 2 cube, 3 sphere), present;
        slot 10 is the kicked sphere.  All zero without ``distractors=True``."""
        return self._sim.get_state(_abi.F_DISTRACTORS)[0].reshape(11, 9).copy()

    def _reset_draws(self):
        # The reference consumes 2 env-RNG uniforms for each of the 10 distractor placements (:62-64) between the
        # button draws and the random init actions; keep the stream aligned.
        x_pos, y_pos = 0.5, 0
        if self._random_target:
            x_pos += 0.15 * self.np_random.uniform(-1, 1)
            y_pos += 0.3 * self.np_random.uniform(-1, 1)
        placements, types = [], []
        with_bodies = getattr(self, "distractors", False)
        for _ in range(10):
            if with_bodies:   # rand_objects[np.random.randint(len(rand_objects))] (:61): the global np.random, untouched when off
                types.append(np.random.randint(3))
            placements.append(0.5 + 0.15 * self.np_random.uniform(-1, 1))
            placements.append(0 + 0.3 * self.np_random.uniform(-1, 1))
        saved, self._random_target = self._random_target, False
        try:
            tail = super(KukaRandButtonGymEnv, self)._reset_draws()[2:]
        finally:
            self._random_target = saved
        draws = [x_pos, y_pos] + tail
        if with_bodies:
            draws += placements + [float(t) for t in types]
        return draws
