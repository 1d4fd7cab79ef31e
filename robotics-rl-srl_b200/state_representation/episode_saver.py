"""
Dataset writer behind ``record_data=True`` -- a from-scratch writer of the on-disk FORMAT the reference's ``EpisodeSaver`` produces
(/root/reference/state_representation/episode_saver.py:139-162 defines the two npz schemas; the env call sites are
kuka_button_gym_env.py:124-126,275-276,362-363 and mobile_robot_env.py:109-111,216-217,274-275).  What is kept is the contract --
constructor keywords, the ``reset`` / ``step`` / ``save`` calls the env classes make, file names, keys, dtypes and row counts -- so that
``environments.dataset_generator`` output stays loadable by the reference's SRL tooling:

    <path><name>/dataset_config.json     {"relative_pos": bool, "max_dist": "<float as str>"}
    <path><name>/env_globals.json        JSON-safe module globals of the env, sorted by key
    <path><name>/preprocessed_data.npz   rewards[S], actions[S(, A)], episode_starts[S] (bool)
    <path><name>/ground_truth.npz        target_positions[E, d], ground_truth_states[S, d], images_path[S] (str)
    <path><name>/record_XXX/             one folder per episode (frames, when an image array is supplied)

with S = recorded transitions and E = episodes: row k of every S-array describes the state an action was taken FROM (the first row of an
episode is the post-reset state, ``episode_starts`` True), and the terminal state of an episode is not recorded.

Internally it is a table writer: rows accumulate in a ``_Table`` of typed columns, an episode is a row range, and the npz files are
re-written from the table whenever an episode closes.  A ``None`` observation contributes its frame NAME only
(``<name>/record_000/frame000000``, the path the reference would have written); an image array is written with cv2, and an already
encoded JPEG file (``bytes``, or a pair of them for two cameras: ``srl_sim.jpeg.encode_jpeg``) is written as it is;
``learn_states`` (the SRL server round trip) is out of scope.
"""
import json
import os

import numpy as np


def _json_safe(value):
    if value is None or isinstance(value, (bool, int, float, str)):
        return True
    if isinstance(value, (list, tuple)):
        return all(_json_safe(v) for v in value)
    if isinstance(value, dict):
        return all(isinstance(k, str) and _json_safe(v) for k, v in value.items())
    return False


def filterJSONSerializableObjects(input_dict):
    """Name kept from the reference's helper (rl_baselines/utils.py:64-75): the JSON-safe entries of a dict, sorted by key."""
    return {k: input_dict[k] for k in sorted(input_dict) if _json_safe(input_dict[k])}


class _Table(object):
    """Append-only columns of equal length."""

    def __init__(self, *names):
        self.cols = {n: [] for n in names}

    def append(self, **row):
        assert set(row) == set(self.cols), "a row fills every column"
        for k, v in row.items():
            self.cols[k].append(v)

    def __len__(self):
        return len(next(iter(self.cols.values())))

    def array(self, name):
        return np.array(self.cols[name])


class EpisodeSaver(object):
    """
    :param name: (str) dataset folder name
    :param max_dist: (float) recorded in dataset_config.json
    :param state_dim: (int) kept for signature compatibility
    :param globals_: (dict) module globals of the env (written to env_globals.json)
    :param learn_every: (int) unused (``learn_states`` is not supported)
    :param learn_states: (bool) must be False
    :param path: (str) prefix of the dataset folder (concatenated, like the reference: 'data/' + name)
    :param relative_pos: (bool) recorded in dataset_config.json
    """

    def __init__(self, name, max_dist, state_dim=-1, globals_=None, learn_every=3, learn_states=False, path='data/', relative_pos=False):
        if learn_states:
            raise NotImplementedError("learn_states (SRL server round trip) is out of scope of the simulator")
        self.name, self.path, self.state_dim = name, path, state_dim
        self.data_folder = path + name
        os.makedirs(self.data_folder, exist_ok=True)
        self.dataset_config = {'relative_pos': relative_pos, 'max_dist': str(max_dist)}
        self._dump_json("dataset_config.json", self.dataset_config)
        if globals_ is not None:
            self._dump_json("env_globals.json", filterJSONSerializableObjects(globals_))
        # one row per recorded transition; `pending` is the state row waiting for the action taken from it
        self._rows = _Table("reward", "action", "episode_start", "state", "frame")
        self._targets = []
        self._pending = None
        self.episode_idx = -1          # public counters the callers read (dataset_generator prints them)
        self.episode_step = 0
        self.n_steps = 0
        self.episode_success = False

    # ---- helpers ------------------------------------------------------------------------------
    def _dump_json(self, fname, obj):
        with open(os.path.join(self.data_folder, fname), "w") as f:
            json.dump(obj, f)

    @property
    def episode_folder(self):
        return "record_{:03d}".format(self.episode_idx)

    def _frame(self, observation):
        """Name of the frame of the current (episode, step); the image itself is written only when an array or encoded JPEG bytes are
        supplied.  ``bytes`` is a finished file (``srl_sim.jpeg.encode_jpeg``), written as ``<frame>.jpg``; a pair of ``bytes`` (two
        cameras) is written as ``<frame>_1.jpg`` and ``<frame>_2.jpg``, the reference's multi-view names."""
        rel = "{}/{}/frame{:06d}".format(self.name, self.episode_folder, self.episode_step)
        if isinstance(observation, bytes) or (isinstance(observation, (tuple, list)) and observation and
                                              all(isinstance(o, bytes) for o in observation)):
            files = [observation] if isinstance(observation, bytes) else list(observation)
            suffixes = [""] if len(files) == 1 else ["_{}".format(i + 1) for i in range(len(files))]
            for data, suffix in zip(files, suffixes):
                with open("{}{}{}.jpg".format(self.path, rel, suffix), "wb") as f:
                    f.write(data)
            return rel
        if observation is not None and getattr(observation, "ndim", 0) == 3:
            import cv2
            cv2.imwrite("{}{}.jpg".format(self.path, rel), cv2.cvtColor(observation[:, :, :3], cv2.COLOR_BGR2RGB))
        return rel

    def _open_state(self, observation, ground_truth, start):
        self._pending = dict(episode_start=start, state=np.array(ground_truth, copy=True), frame=self._frame(observation))

    # ---- calls made by the env classes --------------------------------------------------------
    def reset(self, observation, target_pos, ground_truth):
        """A new episode starts from this state.  A second reset() before any step is ignored (the reference does the same: an env is
        reset once by its constructor's caller and once by the runner)."""
        if self._pending is not None and self._pending["episode_start"]:
            return
        self.episode_idx += 1
        self.episode_step = 0
        self.episode_success = False
        os.makedirs(os.path.join(self.data_folder, self.episode_folder), exist_ok=True)
        self._targets.append(np.array(target_pos, copy=True))
        self._open_state(observation, ground_truth, True)

    def step(self, observation, action, reward, done, ground_truth_state):
        """The action taken from the pending state, its reward, and the state it led to (recorded unless the episode is over)."""
        assert self._pending is not None, "step() before reset()"
        self._rows.append(reward=reward, action=action, **self._pending)
        self._pending = None
        self.episode_step += 1
        self.n_steps += 1
        self.episode_success = self.episode_success or reward > 0
        if done:
            self.save()
        else:
            self._open_state(observation, ground_truth_state, False)

    def save(self):
        """(Re)write both npz files from the rows recorded so far (closed transitions only)."""
        assert len(self._targets) == self.episode_idx + 1
        np.savez(os.path.join(self.data_folder, "preprocessed_data.npz"),
                 rewards=self._rows.array("reward"), actions=self._rows.array("action"), episode_starts=self._rows.array("episode_start"))
        np.savez(os.path.join(self.data_folder, "ground_truth.npz"),
                 target_positions=np.array(self._targets), ground_truth_states=self._rows.array("state"), images_path=self._rows.array("frame"))
