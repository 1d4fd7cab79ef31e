"""
Generate tests/golden/render_hashes_golden.json: SHA-256 hashes of the CPU checker's frames (oracle/liboracle_sim.so, csrc/render_core.h)
for every registered env id, both cameras of its family, at 224 x 224 and 50 x 33, after a fixed seeded rollout.  Frames of scenes
without distractor bodies must never change when the ray caster learns new primitives; tests/test_distractor_frames_cpu.py holds the
checker to these hashes.  Run from a checkout whose oracle is built (`make -C oracle`):

    python tests/golden/gen_render_hashes.py
"""
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (os.path.join(ROOT, "robotics-rl-srl_b200"), ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)

N, T, SEED = 3, 8, 5
SIZES = ((224, 224), (50, 33))
OUT = os.path.join(HERE, "render_hashes_golden.json")


def cases():
    """(env id, cfg, actions [T, N], cameras) of every registered env id."""
    from srl_sim import _abi
    from srl_sim.render import KUKA_CAMERA, KUKA_CAMERA_2, MOBILE_CAMERA, mobile_fpv_camera
    for env_id in sorted(_abi.ENV_KINDS):
        kuka = env_id.startswith("Kuka")
        cfg = dict(seed=SEED, random_target=True)
        if env_id in ("MobileRobot2TargetGymEnv-v0", "MobileRobot1DGymEnv-v0"):
            cfg["is_discrete"] = True
        n_act = 6 if kuka else (2 if env_id == "MobileRobot1DGymEnv-v0" else 4)
        acts = np.random.RandomState(7).randint(0, n_act, size=(T, N)).astype(np.int32)
        cams = [KUKA_CAMERA, KUKA_CAMERA_2] if kuka else [MOBILE_CAMERA, mobile_fpv_camera((2.0, 2.0))]
        yield env_id, cfg, acts, cams


def frame_hashes(backend, env_id, cfg, acts, cams):
    """{"<camera index>/<W>x<H>": [sha256 of each env's frame]} after a reset and a T-step rollout."""
    from srl_sim.model import load_kuka_scene
    from srl_sim.render import camera
    kuka = env_id.startswith("Kuka")
    sim = backend.make_sim(env_id, N, model_blob=load_kuka_scene().blob if kuka else None, **cfg)
    sim.reset(stream=backend.stream())
    obs = backend.zeros((T, N, sim.obs_dim), np.float32); rew = backend.zeros((T, N), np.float32); done = backend.zeros((T, N), np.uint8)
    sim.rollout(T, backend.from_host(acts), None, obs, rew, done, stream=backend.stream())
    out = {}
    for ci, c in enumerate(cams):
        for (w, h) in SIZES:
            buf = backend.zeros((N, h, w, 3), np.uint8)
            sim.render(camera(**c), w, h, buf, stream=backend.stream())
            frames = backend.to_host(buf)
            out["%d/%dx%d" % (ci, w, h)] = [hashlib.sha256(np.ascontiguousarray(frames[k]).tobytes()).hexdigest() for k in range(N)]
    sim.close()
    return out


def main():
    from srl_sim._abi import SimLibrary
    from srl_sim.backend import Backend
    be = Backend(SimLibrary(os.path.join(ROOT, "oracle", "liboracle_sim.so")), -1)
    golden = {env_id: frame_hashes(be, env_id, cfg, acts, cams) for env_id, cfg, acts, cams in cases()}
    with open(OUT, "w") as f:
        json.dump(golden, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote %s (%d env ids)" % (os.path.basename(OUT), len(golden)))


if __name__ == "__main__":
    main()
