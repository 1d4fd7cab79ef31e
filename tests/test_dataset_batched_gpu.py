"""
`python -m environments.dataset_generator --num-envs 64` on the CUDA library against the CUDA `--num-cpu 1` run with the same arguments.
MobileRobot's kernel does the same arithmetic at any batch size, so its arrays are equal.  The Kuka kernel packs envs into warps by
`envs_per_warp` and the lanes of a warp share the contact solver's sweeps, so its float32 trajectories may differ in the last bits between
N = 1 and N = 64: actions, rewards, episode starts and frame names must be equal, states within 1e-3 m.  The frames must decode back to the
scene, and `--distractors` must leave the npz arrays unchanged while changing the frames.
"""
import os

import numpy as np
import pytest

from environments import dataset_generator

pytestmark = pytest.mark.gpu


def _run(tmp, sub, extra):
    root = os.path.join(str(tmp), sub)
    os.makedirs(root, exist_ok=True)
    dataset_generator.main(["--save-path", root + "/", "--name", "ds", "--seed", "5", "-f"] + extra)
    return os.path.join(root, "ds")


def _arrays(d):
    out = {}
    for f in ("preprocessed_data.npz", "ground_truth.npz"):
        z = np.load(os.path.join(d, f))
        out.update({k: z[k] for k in z.files})
    return out


def test_mobile_arrays_equal(tmp_path, cuda_backend):
    args = ["--env", "MobileRobotGymEnv-v0", "-r", "--num-episode", "80"]
    a, b = _arrays(_run(tmp_path, "one", args)), _arrays(_run(tmp_path, "batched", args + ["--num-envs", "64"]))
    assert a.keys() == b.keys()
    for k in a:
        assert np.array_equal(a[k], b[k]), k


def test_kuka_within_float32_tolerance_and_frames_decode(tmp_path, cuda_backend):
    cv2 = pytest.importorskip("cv2")
    args = ["--env", "KukaButtonGymEnv-v0", "--num-episode", "3"]
    one = _arrays(_run(tmp_path, "one", args))
    d = _run(tmp_path, "batched", args + ["--num-envs", "64"])
    bat = _arrays(d)
    for k in ("actions", "rewards", "episode_starts", "images_path"):
        assert np.array_equal(one[k], bat[k]), k
    assert np.abs(one["ground_truth_states"] - bat["ground_truth_states"]).max() < 1e-3
    assert np.abs(one["target_positions"] - bat["target_positions"]).max() < 1e-3
    root = os.path.dirname(d)
    for rel in bat["images_path"][::50]:
        img = cv2.imdecode(np.fromfile(os.path.join(root, rel + ".jpg"), np.uint8), cv2.IMREAD_COLOR)
        assert img.shape == (224, 224, 3) and img.std() > 10        # a drawn scene, not a blank frame


def test_distractors_change_frames_not_arrays(tmp_path, cuda_backend):
    args = ["--env", "KukaRandButtonGymEnv-v0", "--num-episode", "2", "--num-envs", "64"]
    plain, bodies = _run(tmp_path, "plain", args), _run(tmp_path, "bodies", args + ["--distractors"])
    a, b = _arrays(plain), _arrays(bodies)
    for k in a:
        assert np.array_equal(a[k], b[k]), k
    rels = a["images_path"]
    differ = sum(open(os.path.join(os.path.dirname(plain), r + ".jpg"), "rb").read() !=
                 open(os.path.join(os.path.dirname(bodies), r + ".jpg"), "rb").read() for r in rels)
    assert differ > len(rels) // 2
