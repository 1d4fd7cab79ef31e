"""
Mirror of ``python -m environments.dataset_generator`` (environments/dataset_generator.py:37-267): random-agent rollouts of
one registered env, recorded by ``EpisodeSaver`` -- the second consumer of the single-env API (SURVEY.md section 3.5).

Same flags, same per-episode seeding (``seed = RandomState(seed).randint(1e10)``, then one distinct seed per episode,
reference :77-83,169), same output layout, same part fusion (:203-257).  Differences, all forced by what sits underneath:

* the reference forks ``--num-cpu`` OS processes, one PyBullet client each; here every env is an N=1 view on the GPU-resident
  simulator, so the ``num_cpu`` partitions run one after the other in this process and are fused exactly like the
  reference fuses its parts (the episode -> seed assignment is the reference's, so the dataset does not depend on it);
* without ``--num-envs`` the envs run with ``srl_model="ground_truth"``, so frames are recorded by NAME only (``images_path``) and
  no ``.jpg`` is written; the states / targets / actions / rewards are real;
* ``--num-envs N`` (opt-in) records the same episodes WITH their frames: all episodes run on one handle of N envs (``no_auto_reset``;
  finished envs are reset by a masked ``srl_sim_reset`` with the next episode's draws from the env class's own ``_reset_draws``).  Each
  step renders every env (the env's camera, plus the second Kuka camera with ``--multi-view``), encodes the frames as JPEG on the
  device (``srl_sim.jpeg.encode_jpeg``: the bytes ``cv2.imencode`` writes), hands the files to a small writer pool, records the
  ground truth the action is taken from, and steps.  Episode k keeps the seed, the actions (a seeded ``action_space.sample()``) and
  the per-step noise (the env's ``np_random``) the one-partition run gives it, and completed episodes go to one ``EpisodeSaver`` in
  episode order, so the npz / json files equal the ``--num-cpu 1`` output whatever N is (bit for bit on the CPU oracle and for
  MobileRobot; Kuka on CUDA: see ``batched_run``).  Kuka2Button and MobileRobot2Target keep extra per-episode state in their env
  objects and are not supported in this mode;
* ``--run-ppo2`` (a CnnPolicy on pixels) and ``--display`` are not available.
"""
import argparse
import glob
import os
import shutil
import time

import numpy as np

from environments.registry import registered_env


def convertImagePath(args, path, record_id_start):
    """
    Used to convert an image path, from one location, to another (reference :23-34)
    """
    image_name = path.split("/")[-1]
    new_record_id = record_id_start + int(path.split("/")[-2].split("_")[-1])
    return args.name + "/record_{:03d}".format(new_record_id) + "/" + image_name


def env_thread(args, thread_num, partition=True):
    """
    Run a session of an environment (reference :37-121, random-agent branch)
    :param args: (ArgumentParser object)
    :param thread_num: (int) The partition ID of the environment session
    :param partition: (bool) If the output should be in multiple parts (default=True)
    """
    # the env records / returns the ground-truth state and no frames (the reference's default here is raw_pixels, whose frames this
    # generator only ever hands to EpisodeSaver); --num-envs records the frames too (batched_run)
    env = registered_env[args.env][0](**_env_kwargs(args, args.name + "_part-" + str(thread_num) if partition else args.name))
    frames = 0
    start_time = time.time()
    # divide evenly, then do an extra one for only some of them in order to get the right count
    for i_episode in range(args.num_episode // args.num_cpu + 1 * (args.num_episode % args.num_cpu > thread_num)):
        # seed + position in this slice + size of slice (with reminder if uneven partitions)
        seed = args.seed + i_episode + args.num_episode // args.num_cpu * thread_num + \
            (thread_num if thread_num <= args.num_episode % args.num_cpu else args.num_episode % args.num_cpu)
        env.seed(seed)
        env.action_space.seed(seed)  # this is for the sample() function from gym.space
        env.reset()
        done = False
        t = 0
        while not done:
            _, _, done, _ = env.step(env.action_space.sample())
            frames += 1
            t += 1
            if done and args.verbose:
                print("Episode finished after {} timesteps".format(t + 1))
    if args.verbose:
        print("part {}: {:.2f} FPS".format(thread_num, frames / max(1e-9, time.time() - start_time)))
    env.close()
    return frames


BATCHED_UNSUPPORTED = ("Kuka2ButtonGymEnv-v0", "MobileRobot2TargetGymEnv-v0")


def _env_kwargs(args, name, srl_model="ground_truth"):
    kw = {
        "max_distance": args.max_distance,
        "random_target": args.random_target,
        "force_down": True,
        "is_discrete": not args.continuous_actions,
        "renders": False,
        "record_data": not args.no_record_data,
        "multi_view": args.multi_view,
        "save_path": args.save_path,
        "shape_reward": args.shape_reward,
        "srl_model": srl_model,
        "name": name,
    }
    if args.distractors:
        kw["distractors"] = True
    return kw


def batched_run(args):
    """
    ``--num-envs N``: every episode on one handle of N envs, frames rendered and JPEG-encoded on the device.

    The env class is instantiated once (with ``record_data``: its ``EpisodeSaver`` is the one the one-partition run writes through) and
    serves as the source of everything per episode the class defines: the seeded ``np_random`` and action space, ``_reset_draws``, the
    ground-truth / target accessors and the simulator configuration.  Only its saver and its methods are used; its own N = 1 handle
    stays idle.  Per env slot the generator keeps the episode's RNG and action space, so episode k consumes them exactly as
    ``env.seed(seed); env.action_space.seed(seed); env.reset(); env.step(env.action_space.sample()) ...`` does.

    Results: on the CPU oracle and for MobileRobot (whose arithmetic does not depend on the batch) the npz files are bit-identical to
    ``--num-cpu 1``.  The Kuka CUDA kernel packs envs into warps by ``envs_per_warp`` (0 = chosen from N), and the lanes of a warp
    share the sweeps of the contact solver, so a Kuka env's float32 trajectory may differ in the last bits between N = 1 and N = 64;
    actions, rewards, episode starts and frame names stay equal and the states within 1e-3 m (tests/test_dataset_batched_gpu.py).
    :return: (int) recorded frames
    """
    import copy
    from concurrent.futures import ThreadPoolExecutor

    from srl_sim import _abi
    from srl_sim.jpeg import encode_jpeg, release_buffers
    from srl_sim.render import KUKA_CAMERA, KUKA_CAMERA_2, MOBILE_CAMERA, render_batch

    if args.env in BATCHED_UNSUPPORTED:
        raise ValueError("--num-envs does not support %s (its env object keeps per-episode state the batch does not restate)" % args.env)
    env = registered_env[args.env][0](**_env_kwargs(args, args.name))
    kuka = args.env.startswith("Kuka")
    be = env._backend
    cfg = {name: getattr(env._sim.cfg, name) for name, _ in _abi.SrlCfg._fields_ if name != "struct_size"}
    n_envs = args.num_envs             # the batch layout is N's even while fewer episodes remain (idle envs step unrecorded)
    sim = be.make_sim(args.env, n_envs, seed=0, model_blob=getattr(env._sim, "_blob", None), **cfg)
    if getattr(env, "distractors", False):
        sim.set_distractors(env._sim._dist_blob)
    if kuka:
        from environments.kuka_gym import kuka_button_gym_env as kmod
        noise_std = kmod.NOISE_STD if env._is_discrete else kmod.NOISE_STD_CONTINUOUS
        cams = [KUKA_CAMERA, KUKA_CAMERA_2] if args.multi_view else [KUKA_CAMERA]
    else:
        from environments.mobile_robot import mobile_robot_env as mmod
        noise_std = mmod.NOISE_STD
        cams = [dict(MOBILE_CAMERA, target=env.camera_target_pos)]
    record = not args.no_record_data
    saver = env.saver

    def accessors(robot, target):
        """The env class's own getGroundTruth / getTargetPos on one env's state."""
        if kuka:
            env._arm_pos, env.button_pos = robot, target
        else:
            env.robot_pos, env.target_pos = robot, target
        return np.array(env.getGroundTruth(), copy=True), np.array(env.getTargetPos(), copy=True)

    slot_episode = [-1] * n_envs        # episode index run by each slot (-1: idle)
    slot_rng, slot_space = [None] * n_envs, [None] * n_envs
    episodes = {}                       # k -> dict(target, rows=[(state, action, reward, done)], state)
    next_k, next_flush, frames_done = 0, 0, 0

    def start(slots):
        nonlocal next_k
        mask = np.zeros(n_envs, np.uint8)
        rows = None
        for i in slots:
            if next_k >= args.num_episode:
                slot_episode[i] = -1
                continue
            seed = args.seed + next_k
            env.seed(seed)
            space = copy.deepcopy(env.action_space)
            space.seed(seed)
            draws = env._reset_draws()
            if rows is None:
                rows = np.zeros((n_envs, len(draws)), np.float64)
            rows[i] = draws
            slot_episode[i], slot_rng[i], slot_space[i] = next_k, env.np_random, space
            episodes[next_k] = dict(rows=[], t=0)
            mask[i] = 1
            next_k += 1
        if mask.any():
            sim.reset(mask=be.from_host(mask), reset_draws=be.from_host(rows), stream=be.stream())
        return mask

    def flush():
        nonlocal next_flush
        while next_flush in episodes and episodes[next_flush].get("closed"):
            ep = episodes.pop(next_flush)
            if record:
                saver.reset(None, ep["target"], ep["rows"][0][0])
                for j, (_, action, reward, done) in enumerate(ep["rows"]):
                    nxt = ep["rows"][j + 1][0] if j + 1 < len(ep["rows"]) else ep["last"]
                    saver.step(None, action, reward, done, nxt)
            next_flush += 1

    is_discrete = env._is_discrete
    act_shape = (n_envs,) if is_discrete else (n_envs, sim.action_dim)
    obs = be.zeros((n_envs, sim.obs_dim), np.float32)
    rew = be.zeros((n_envs,), np.float32)
    done = be.zeros((n_envs,), np.uint8)
    start(range(n_envs))
    fresh = [True] * n_envs
    pool = ThreadPoolExecutor(max_workers=4)
    pending = []
    start_time = time.time()

    def write(path, data):
        with open(path, "wb") as f:
            f.write(data)

    while any(k >= 0 for k in slot_episode):
        robot, target = sim.get_state(_abi.F_ROBOT_POS), sim.get_state(_abi.F_TARGET_POS)
        active = [i for i in range(n_envs) if slot_episode[i] >= 0]
        if record:
            frames = render_batch(sim, be, cams)
            files = [encode_jpeg(be, frames, quality=args.quality, channel_offset=3 * c) for c in range(len(cams))]
        acts = np.zeros(act_shape, np.int32 if is_discrete else np.float32)
        noise = np.zeros(n_envs, np.float32)
        chosen = {}
        for i in active:
            k = slot_episode[i]
            ep = episodes[k]
            gt, tgt = accessors(robot[i].copy(), target[i].copy())
            if fresh[i]:
                ep["target"], fresh[i] = tgt, False
                if record:
                    os.makedirs(os.path.join(args.save_path + args.name, "record_{:03d}".format(k)), exist_ok=True)
            if record:
                base = os.path.join(args.save_path + args.name, "record_{:03d}".format(k), "frame{:06d}".format(ep["t"]))
                if len(cams) == 1:
                    pending.append(pool.submit(write, base + ".jpg", files[0][i]))
                else:
                    for c in range(len(cams)):
                        pending.append(pool.submit(write, base + "_{}.jpg".format(c + 1), files[c][i]))
            action = slot_space[i].sample()
            chosen[i] = (gt, action)
            acts[i] = int(action) if is_discrete else np.asarray(action, np.float32).reshape(-1)
            noise[i] = slot_rng[i].normal(0.0, scale=noise_std)
        sim.step(be.from_host(acts), noise=be.from_host(noise), obs_out=obs, rew_out=rew, done_out=done, stream=be.stream())
        r_host, d_host = be.to_host(rew), be.to_host(done)
        robot_next = sim.get_state(_abi.F_ROBOT_POS)
        finished = []
        for i in active:
            ep = episodes[slot_episode[i]]
            r = float(r_host[i])
            reward = r if args.shape_reward else int(r)
            d = bool(d_host[i])
            gt, action = chosen[i]
            ep["rows"].append((gt, action, reward, d))
            ep["t"] += 1
            frames_done += 1
            if d:
                ep["last"] = accessors(robot_next[i].copy(), target[i].copy())[0]
                ep["closed"] = True
                finished.append(i)
                if args.verbose:
                    print("Episode finished after {} timesteps".format(ep["t"] + 1))
        if finished:
            for i in finished:
                fresh[i] = True
            start(finished)
            flush()
        if len(pending) > 4096:
            for p in pending:
                p.result()
            pending = []
    for p in pending:
        p.result()
    pool.shutdown()
    flush()
    release_buffers()
    if args.verbose:
        print("{} envs: {:.2f} FPS".format(n_envs, frames_done / max(1e-9, time.time() - start_time)))
    sim.close()
    env.close()
    return frames_done


def fuse_parts(args):
    """The reference's part fusion (:203-257)."""
    file_parts = sorted(glob.glob(args.save_path + args.name + "_part-[0-9]*"), key=lambda a: int(a.split("-")[-1]))
    os.rename(file_parts[0] + "/dataset_config.json", args.save_path + args.name + "/dataset_config.json")
    os.rename(file_parts[0] + "/env_globals.json", args.save_path + args.name + "/env_globals.json")
    ground_truth, preprocessed_data = None, None
    record_id = 0
    for part in file_parts:
        records = sorted(glob.glob(part + "/record_[0-9]*"), key=lambda a: int(a.split("_")[-1]))
        record_id_start = record_id
        for record in records:
            os.renames(record, args.save_path + args.name + "/record_{:03d}".format(record_id))
            record_id += 1
        ground_truth_load = np.load(part + "/ground_truth.npz")
        preprocessed_data_load = np.load(part + "/preprocessed_data.npz")
        gt = {arr: (np.array([convertImagePath(args, path, record_id_start) for path in ground_truth_load[arr]])
                    if arr == "images_path" else ground_truth_load[arr]) for arr in ground_truth_load.files}
        pd = {arr: preprocessed_data_load[arr] for arr in preprocessed_data_load.files}
        if ground_truth is None:
            ground_truth, preprocessed_data = gt, pd
        else:
            ground_truth = {k: np.concatenate((ground_truth[k], gt[k])) for k in gt}
            preprocessed_data = {k: np.concatenate((preprocessed_data[k], pd[k])) for k in pd}
        shutil.rmtree(part, ignore_errors=True)
    np.savez(args.save_path + args.name + "/ground_truth.npz", **ground_truth)
    np.savez(args.save_path + args.name + "/preprocessed_data.npz", **preprocessed_data)


def main(argv=None):
    parser = argparse.ArgumentParser(description='Deteministic dataset generator for SRL training ' +
                                                 '(can be used for environment testing)')
    parser.add_argument('--num-cpu', type=int, default=1, help='number of partitions (the reference: processes)')
    parser.add_argument('--num-episode', type=int, default=50, help='number of episode to run')
    parser.add_argument('--save-path', type=str, default='srl_zoo/data/', help='Folder where the environments will save the output')
    parser.add_argument('--name', type=str, default='kuka_button', help='Folder name for the output')
    parser.add_argument('--env', type=str, default='KukaButtonGymEnv-v0', help='The environment wanted', choices=list(registered_env.keys()))
    parser.add_argument('--no-record-data', action='store_true', default=False)
    parser.add_argument('--max-distance', type=float, default=0.28, help='Beyond this distance from the goal, the agent gets a negative reward')
    parser.add_argument('-c', '--continuous-actions', action='store_true', default=False)
    parser.add_argument('--seed', type=int, default=0, help='the seed')
    parser.add_argument('-f', '--force', action='store_true', default=False, help='Force the save, even if it overrides something else')
    parser.add_argument('-r', '--random-target', action='store_true', default=False, help='Set the button to a random position')
    parser.add_argument('--multi-view', action='store_true', default=False,
                        help='Kuka: record the second camera too (with --num-envs: frameXXXXXX_1.jpg / _2.jpg)')
    parser.add_argument('--num-envs', type=int, default=0,
                        help='run every episode on one batched handle of N envs and record the frames as .jpg (encoded on the device)')
    parser.add_argument('--quality', type=int, default=95, help='JPEG quality of the recorded frames (--num-envs), as cv2.IMWRITE_JPEG_QUALITY')
    parser.add_argument('--distractors', action='store_true', default=False,
                        help='KukaRandButtonGymEnv-v0: simulate and draw the random objects and the kicked sphere')
    parser.add_argument('--shape-reward', action='store_true', default=False, help='Shape the reward (reward = - distance) instead of a sparse reward')
    parser.add_argument('--reward-dist', action='store_true', default=False, help='Prints out the reward distribution when the dataset generation is finished')
    parser.add_argument('--verbose', action='store_true', default=False)
    args = parser.parse_args(argv)

    assert (args.num_cpu > 0), "Error: number of cpu must be positive and non zero"
    assert (args.max_distance > 0), "Error: max distance must be positive and non zero"
    assert (args.num_episode > 0), "Error: number of episodes must be positive and non zero"
    assert not args.reward_dist or not args.shape_reward, "Error: cannot display the reward distribution for continuous reward"
    assert args.num_envs >= 0, "Error: --num-envs must be positive"
    assert not (args.num_envs and args.num_cpu > 1), "Error: --num-envs runs every episode on one handle; it excludes --num-cpu > 1"
    assert 1 <= args.quality <= 100, "Error: --quality must be in 1..100"
    assert not args.distractors or args.env == "KukaRandButtonGymEnv-v0", "Error: --distractors is only available for KukaRandButtonGymEnv-v0"
    if args.num_cpu > args.num_episode:
        args.num_cpu = args.num_episode
    # this is done so seed 0 and 1 are different and not simply offset of the same datasets.
    args.seed = np.random.RandomState(args.seed).randint(int(1e10))
    if not args.no_record_data and os.path.exists(args.save_path + args.name):
        assert args.force, "Error: save directory '{}' already exists".format(args.save_path + args.name)
        shutil.rmtree(args.save_path + args.name)
        for part in glob.glob(args.save_path + args.name + "_part-[0-9]*"):
            shutil.rmtree(part)
    if not args.no_record_data:
        os.makedirs(args.save_path + args.name)
    if args.num_envs:
        frames = batched_run(args)
    elif args.num_cpu == 1:
        frames = env_thread(args, 0, partition=False)
    else:
        frames = sum(env_thread(args, i, partition=True) for i in range(args.num_cpu))
    if not args.no_record_data and args.num_cpu > 1:
        fuse_parts(args)
    if args.reward_dist:
        rewards, counts = np.unique(np.load(args.save_path + args.name + "/preprocessed_data.npz")['rewards'], return_counts=True)
        counts = ["{:.2f}%".format(val * 100) for val in counts / np.sum(counts)]
        print("reward distribution:")
        [print(" ", reward, count) for reward, count in list(zip(rewards, counts))]
    return frames


if __name__ == '__main__':
    main()
