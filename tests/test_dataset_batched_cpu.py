"""
`python -m environments.dataset_generator --num-envs N` on the CPU oracle: every episode on one batched handle, frames rendered and
JPEG-encoded (the CPU checker of include/srl_image.h), against the one-partition run (`--num-cpu 1`) with the same arguments.  The npz and
json files must be the same bytes, every `images_path` entry must have its .jpg, and each file must be what cv2 writes for the frame of
that recorded state -- here the frame the single env renders itself (`srl_model="raw_pixels"`, `record_data=True`, which writes its frames
with cv2.imwrite) when replaying the same seeds.
"""
import os

import numpy as np
import pytest

from environments import dataset_generator

cv2 = pytest.importorskip("cv2")

FILES = ("preprocessed_data.npz", "ground_truth.npz", "dataset_config.json", "env_globals.json")


def _run(tmp, sub, extra, name="ds"):
    root = os.path.join(str(tmp), sub)
    os.makedirs(root, exist_ok=True)
    dataset_generator.main(["--save-path", root + "/", "--name", name, "--seed", "3", "-f"] + extra)
    return os.path.join(root, name)


def _same_files(a, b):
    for f in FILES:
        assert open(os.path.join(a, f), "rb").read() == open(os.path.join(b, f), "rb").read(), f


def _replay_frames(tmp, env_id, n_episodes, extra_kwargs):
    """The single env with raw_pixels observations, driven like the one-partition generator: its saver writes cv2's file per state."""
    from environments.registry import registered_env
    seed = np.random.RandomState(3).randint(int(1e10))
    env = registered_env[env_id][0](srl_model="raw_pixels", record_data=True, name="replay", save_path=str(tmp) + "/", force_down=True,
                                    renders=False, **extra_kwargs)
    for k in range(n_episodes):
        env.seed(seed + k)
        env.action_space.seed(seed + k)
        env.reset()
        done = False
        while not done:
            _, _, done, _ = env.step(env.action_space.sample())
    env.close()
    return os.path.join(str(tmp), "replay")


def _check_frames(dataset, replay, name):
    gt = np.load(os.path.join(dataset, "ground_truth.npz"))
    assert len(gt["images_path"]) > 0
    for rel in gt["images_path"]:
        ours = open(os.path.join(os.path.dirname(dataset), rel + ".jpg"), "rb").read()
        theirs = open(os.path.join(replay, rel[len(name) + 1:] + ".jpg"), "rb").read()
        assert ours == theirs, rel


@pytest.mark.parametrize("env_id, extra, kwargs, n_episodes", [
    ("MobileRobotGymEnv-v0", ["-r"], dict(random_target=True), 3),
    ("KukaButtonGymEnv-v0", [], dict(), 2),
])
def test_batched_generator_reproduces_one_partition(tmp_path, use_oracle_backend, env_id, extra, kwargs, n_episodes):
    args = ["--env", env_id, "--num-episode", str(n_episodes)] + extra
    one = _run(tmp_path, "one", args + ["--num-cpu", "1"])
    batched = _run(tmp_path, "batched", args + ["--num-envs", "2"])
    for f in FILES:
        assert os.path.isfile(os.path.join(batched, f))
    _same_files(one, batched)
    starts = np.load(os.path.join(batched, "preprocessed_data.npz"))["episode_starts"]
    assert starts.sum() == n_episodes
    _check_frames(batched, _replay_frames(tmp_path, env_id, n_episodes, kwargs), "ds")


def test_batched_generator_multi_view_writes_both_cameras(tmp_path, use_oracle_backend):
    d = _run(tmp_path, "mv", ["--env", "KukaButtonGymEnv-v0", "--num-episode", "1", "--num-envs", "2", "--multi-view"])
    gt = np.load(os.path.join(d, "ground_truth.npz"))
    root = os.path.dirname(d)
    for rel in gt["images_path"]:
        a = open(os.path.join(root, rel + "_1.jpg"), "rb").read()
        b = open(os.path.join(root, rel + "_2.jpg"), "rb").read()
        assert a[:2] == b"\xff\xd8" and b[:2] == b"\xff\xd8" and a != b
        assert not os.path.exists(os.path.join(root, rel + ".jpg"))


def test_num_envs_with_num_cpu_is_an_error(tmp_path):
    with pytest.raises(AssertionError):
        _run(tmp_path, "x", ["--num-envs", "2", "--num-cpu", "2"])
