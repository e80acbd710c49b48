"""LIBERO action-inference wrapper -- mirror of reference utils/eval_utils_libero.py:43-179 (`ModelWrapper.step`), without the
MuJoCo simulator (out of scope).  Images are raw uint8 camera frames or already-preprocessed tensors (see `ModelWrapper.step`).

What differs from the CALVIN wrapper (utils/eval_utils_calvin.py here), all kept from the reference:
  * state = [eef_pos(3), euler_xyz(eef_quat)(3), g] with g = the gripper command of the PREVIOUS action (initially -1), or
    with `gripper_width` the two finger joint positions `robot0_gripper_qpos` -> an 8-dim state (:112-115);
  * temporal ensembling (`--eval_libero_ensembling`, :159-176): every step's `action_pred_steps` predictions are written
    into `all_time_actions[t, t:t+steps]`, the action for step t is the exp(-k*i)-weighted mean (oldest first, k =
    `ensembling_temp`) over all populated predictions for t, then the gripper channel is thresholded at 0.5 -> {-1, +1};
  * `self.gripper_state` is fed back from the returned action (:178).
Without ensembling the reference's `step` never assigns `action` (UnboundLocalError at :178); here that case selects the
window row like the CALVIN wrapper does (utils/eval_utils_calvin.py:138-145), which is what the authors' CALVIN loop does.
"""
from __future__ import annotations

import numpy as np
import torch

from .eval_utils_calvin import BatchedRolloutEngine, RolloutEngine


def quaternion_to_euler(q):
    """scipy `Rotation.from_quat(q).as_euler('xyz')` (reference :30-34): q = (x, y, z, w), extrinsic x-y-z angles in radians."""
    x, y, z, w = (float(v) for v in q)
    n = (x * x + y * y + z * z + w * w) ** 0.5
    x, y, z, w = x / n, y / n, z / n, w / n
    roll = np.arctan2(2.0 * (w * x + y * z), 1.0 - 2.0 * (x * x + y * y))
    pitch = np.arcsin(np.clip(2.0 * (w * y - z * x), -1.0, 1.0))
    yaw = np.arctan2(2.0 * (w * z + x * y), 1.0 - 2.0 * (y * y + z * z))
    return np.array([roll, pitch, yaw])


class ModelWrapper(RolloutEngine):
    def __init__(self, model, cast_dtype=torch.bfloat16, history_len=7, use_ensembling=False, ensembling_temp=0.01,
                 libero_eval_max_steps=600, action_pred_steps=3, gripper_width=False, device="cuda", use_cuda_graph=True,
                 incremental=False, prune=True):
        super().__init__(model, cast_dtype, history_len, action_pred_steps, device, use_cuda_graph, incremental, prune,
                         state_dim=8 if gripper_width else 7)
        self.use_ensembling = use_ensembling
        self.ensembling_temp = ensembling_temp
        self.libero_eval_max_steps = libero_eval_max_steps
        self.gripper_width = gripper_width
        self.cnt = 0
        self.gripper_state = np.array([-1.0])
        self.all_time_actions = None
        if self.use_ensembling:
            self._alloc_ensemble()

    def _alloc_ensemble(self):
        self.all_time_actions = torch.zeros([self.libero_eval_max_steps, self.libero_eval_max_steps + self.action_pred_steps, 7],
                                            device=self.device)

    def reset(self):                                                        # :80-92
        self.reset_window()
        self.gripper_state = np.array([-1.0])
        if self.use_ensembling:
            self._alloc_ensemble()
        self.cnt += 1

    def build_state(self, eef_pos, eef_quat, gripper_qpos=None):
        """:106-115 -> float64 numpy [7] or [8]."""
        pos, ori = np.asarray(eef_pos, dtype=np.float64), quaternion_to_euler(eef_quat)
        if not self.gripper_width:
            return np.concatenate([pos, ori, self.gripper_state])
        return np.concatenate([pos, ori, np.asarray(gripper_qpos, dtype=np.float64)])

    @torch.no_grad()
    def step(self, image_agentview, image_eye_in_hand, eef_pos, eef_quat, gripper_qpos, text_tokens, timestep, sample_noise=None):
        """One env step -> action [7] numpy; see module docstring.  image_* are the raw uint8 [h, w, 3] camera frames
        (`obs["agentview_image"]`, `obs["robot0_eye_in_hand_image"]`) or [3,224,224] preprocessed tensors.  A raw agent view
        is flipped vertically before preprocessing, as the reference does (:96); a preprocessed one is taken as it is."""
        state = torch.from_numpy(self.build_state(eef_pos, eef_quat, gripper_qpos))
        arm, gripper, _ = self.infer(image_agentview, image_eye_in_hand, state, text_tokens, sample_noise, flip_static=True)
        if self.use_ensembling:
            action = torch.cat((arm, gripper), dim=-1).unsqueeze(0)           # (1, action_pred_steps, 7)   :165
            self.all_time_actions[timestep:timestep + 1, timestep:timestep + self.action_pred_steps] = action.to(self.all_time_actions.dtype)
            cur = self.all_time_actions[:, timestep]
            cur = cur[torch.all(cur != 0, dim=1)]
            w = np.exp(-self.ensembling_temp * np.arange(len(cur)))
            w = torch.from_numpy(w / w.sum()).to(self.device).unsqueeze(1)
            act = (cur * w).sum(dim=0, keepdim=True)
            act = torch.cat((act[:, :6], (act[:, 6:] > 0.5).to(act.dtype)), dim=-1)
            act[:, -1] = (act[:, -1] - 0.5) * 2
            action = act.detach().cpu().numpy()[-1]
        else:
            act = torch.cat((arm[0].float(), (gripper[0] > 0.5).float()), dim=-1)
            act[-1] = (act[-1] - 0.5) * 2
            action = act.to(torch.float16).cpu().numpy()
        self.gripper_state = np.array([float(action[-1])])                    # :178
        return action


class BatchedModelWrapper(BatchedRolloutEngine):
    """LIBERO rollout wrapper for `num_envs` environments: `ModelWrapper.step` per env, batched (see BatchedRolloutEngine).
    Per env: the agent-view flip, the 7- or 8-dim (`gripper_width`) state, the gripper command fed back from the previous
    action and the temporal-ensembling buffer."""

    def __init__(self, model, num_envs, cast_dtype=torch.bfloat16, history_len=7, use_ensembling=False, ensembling_temp=0.01,
                 libero_eval_max_steps=600, action_pred_steps=3, gripper_width=False, device="cuda", use_cuda_graph=True,
                 incremental=True):
        super().__init__(model, num_envs, cast_dtype, history_len, action_pred_steps, device, use_cuda_graph, incremental,
                         state_dim=8 if gripper_width else 7)
        self.use_ensembling = use_ensembling
        self.ensembling_temp = ensembling_temp
        self.libero_eval_max_steps = libero_eval_max_steps
        self.gripper_width = gripper_width
        self.gripper_state = [np.array([-1.0]) for _ in range(num_envs)]
        self.all_time_actions = [self._ensemble_buffer() if use_ensembling else None for _ in range(num_envs)]

    def _ensemble_buffer(self):
        return torch.zeros([self.libero_eval_max_steps, self.libero_eval_max_steps + self.action_pred_steps, 7],
                           device=self.device)

    def reset(self, env):                                                   # :80-92
        self.reset_window(env)
        self.gripper_state[env] = np.array([-1.0])
        if self.use_ensembling:
            self.all_time_actions[env] = self._ensemble_buffer()

    def build_state(self, env, eef_pos, eef_quat, gripper_qpos=None):
        pos, ori = np.asarray(eef_pos, dtype=np.float64), quaternion_to_euler(eef_quat)
        if not self.gripper_width:
            return np.concatenate([pos, ori, self.gripper_state[env]])
        return np.concatenate([pos, ori, np.asarray(gripper_qpos, dtype=np.float64)])

    @torch.no_grad()
    def step(self, envs, image_agentview, image_eye_in_hand, eef_pos, eef_quat, gripper_qpos, text_tokens, timesteps,
             sample_noise=None):
        """One env step for each env in `envs` -> actions [n, 7] numpy (see ModelWrapper.step; per-env arguments stacked or
        listed in the order of `envs`, gripper_qpos may be None without gripper_width)."""
        n = len(envs)
        qpos = gripper_qpos if gripper_qpos is not None else [None] * n
        state = torch.from_numpy(np.stack([self.build_state(e, eef_pos[i], eef_quat[i], qpos[i]) for i, e in enumerate(envs)]))
        arm, gripper, _ = self.infer_batch(envs, image_agentview, image_eye_in_hand, state, text_tokens, sample_noise,
                                           flip_static=True)
        actions = []
        for i, e in enumerate(envs):
            t = int(timesteps[i])
            if self.use_ensembling:
                buf = self.all_time_actions[e]
                action = torch.cat((arm[i], gripper[i]), dim=-1).unsqueeze(0)        # (1, action_pred_steps, 7)   :165
                buf[t:t + 1, t:t + self.action_pred_steps] = action.to(buf.dtype)
                cur = buf[:, t]
                cur = cur[torch.all(cur != 0, dim=1)]
                w = np.exp(-self.ensembling_temp * np.arange(len(cur)))
                w = torch.from_numpy(w / w.sum()).to(self.device).unsqueeze(1)
                act = (cur * w).sum(dim=0, keepdim=True)
                act = torch.cat((act[:, :6], (act[:, 6:] > 0.5).to(act.dtype)), dim=-1)
                act[:, -1] = (act[:, -1] - 0.5) * 2
                a = act.detach().cpu().numpy()[-1]
            else:
                act = torch.cat((arm[i, 0].float(), (gripper[i, 0] > 0.5).float()), dim=-1)
                act[-1] = (act[-1] - 0.5) * 2
                a = act.to(torch.float16).cpu().numpy()
            self.gripper_state[e] = np.array([float(a[-1])])                     # :178
            actions.append(a)
        return np.stack(actions)
