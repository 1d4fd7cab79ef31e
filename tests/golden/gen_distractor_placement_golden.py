"""
Generate tests/golden/distractor_placement_golden.npz by running the REFERENCE KukaRandButtonGymEnv
(/root/reference/environments/kuka_gym/kuka_rand_button_gym_env.py -- unmodified) on tests/golden/fake_pybullet.py and recording
where its reset() loads the distractor objects and the sphere (fake_pybullet.loadURDF is wrapped, the file itself is not edited).
Build container only:

    python tests/golden/gen_distractor_placement_golden.py

Per case (seed, random_target, global np.random seed): 3 consecutive resets; per reset the button position and every loaded
object / sphere as (type index, x, y, z), type 0 duck_vhacd, 1 lego, 2 cube_small, 3 sphere_small, in load order.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
import _ref_stubs  # noqa: E402
import fake_pybullet  # noqa: E402

_ref_stubs.install(os.path.join(ROOT, "robotics-rl-srl_b200"), real_pybullet=False)
sys.modules["pybullet"] = fake_pybullet.as_module()
import torch  # noqa: E402,F401  (the reference imports it)

from environments.kuka_gym.kuka_rand_button_gym_env import KukaRandButtonGymEnv  # noqa: E402

assert _ref_stubs.REFERENCE_ROOT in sys.modules[KukaRandButtonGymEnv.__module__].__file__, "must import the reference class"

TYPES = {"duck_vhacd.urdf": 0, "lego.urdf": 1, "cube_small.urdf": 2, "sphere_small.urdf": 3}
CASES = [(0, False, 100), (1, True, 101), (2, True, 102), (3, False, 103), (4, True, 104), (5, False, 105)]   # seed, random_target, np seed
RESETS = 3

loaded = []
_load = fake_pybullet.loadURDF


def _recording_load(path, *args, **kwargs):
    name = os.path.basename(str(path))
    if name in TYPES:
        pos = args[0] if args else kwargs.get("basePosition")
        loaded.append([TYPES[name], float(pos[0]), float(pos[1]), float(pos[2])])
    return _load(path, *args, **kwargs)


def main():
    sys.modules["pybullet"].loadURDF = _recording_load
    out = {}
    for c, (seed, random_target, np_seed) in enumerate(CASES):
        env = KukaRandButtonGymEnv(srl_model="ground_truth", is_discrete=True, random_target=random_target)
        env.seed(seed)
        np.random.seed(np_seed)
        bodies, buttons = [], []
        for _ in range(RESETS):
            del loaded[:]
            env.reset()
            bodies.append(np.asarray(loaded, np.float64).reshape(-1, 4))
            buttons.append(np.array(env.button_pos[:2], np.float64))
        out["case%d/params" % c] = np.array([seed, int(random_target), np_seed], np.int64)
        out["case%d/counts" % c] = np.array([len(b) for b in bodies], np.int64)
        out["case%d/bodies" % c] = np.concatenate(bodies, axis=0)
        out["case%d/button_xy" % c] = np.stack(buttons)
        print("case", c, "bodies per reset", [len(b) for b in bodies])
    np.savez_compressed(os.path.join(HERE, "distractor_placement_golden.npz"), **out)
    print("wrote distractor_placement_golden.npz")


if __name__ == "__main__":
    main()
