"""Action-inference wrapper -- mirror of reference utils/eval_utils_calvin.py:48-147 (`ModelWrapper.step`), without the
simulator (out of scope).  Images are raw uint8 camera frames (CLIP's image transform then runs on the device) or
already-preprocessed tensors; tokenisation is data-side.

Semantics kept (reference :107-145): growing-then-sliding window of `history_len` frames, window padded by repeating the
last frame, the instruction tokens of the FIRST step frozen for the episode and repeated over the window, gripper
thresholding at 0.5 and rescale to {-1, +1}, selection of row `num_step-1` (the last row once the window is full), fp16
numpy action.

Two execution modes:
  * incremental=False -- what the reference does: a full-window `mode='test'` forward every env step (ViT on 2*S frames,
    resampler, backbone on all L tokens, DDIM for all S timesteps, S-1 of which are discarded), replayed as ONE CUDA graph.
  * incremental=True  -- rollout-level incremental inference (SURVEY §8 f-1): each frame's position-independent token block
    (ViT + resampler + projectors + state encoder) is computed ONCE when the frame arrives and kept in the window, the text
    slot once per episode; an env step then runs the backbone and the DDIM sampler for the selected timestep only
    (`DreamVLA.rollout_action`).  `prune=False` keeps all L backbone tokens (activations of the selected rows are those of
    the full-window forward); `prune=True` also drops the tokens no selected row can attend to.
"""
from __future__ import annotations

from collections import deque

import numpy as np
import torch

from .data_utils import preprocess_image


class RolloutEngine:
    """Window bookkeeping + CUDA-graph replay shared by the CALVIN and LIBERO wrappers."""

    def __init__(self, model, cast_dtype=torch.bfloat16, history_len=10, action_pred_steps=3, device="cuda",
                 use_cuda_graph=True, incremental=False, prune=True, state_dim=7):
        self.model = model.module if hasattr(model, "module") else model
        self.cast_type = cast_dtype
        self.history_len = history_len
        self.action_pred_steps = action_pred_steps
        self.device = device
        self.use_cuda_graph = use_cuda_graph
        self.incremental = incremental
        self.prune = prune
        self.state_dim = state_dim
        self._graph = None            # full-window graph
        self._enc_graph = None        # incremental: one-frame encoder graph
        self._act_graphs = {}         # incremental: selected timestep -> action graph
        self.reset_window()

    # ---- window ----------------------------------------------------------------------------------------------------
    def reset_window(self):
        self.img_queue = deque(maxlen=self.history_len)
        self.gripper_queue = deque(maxlen=self.history_len)
        self.state_queue = deque(maxlen=self.history_len)
        self.tok_queue = deque(maxlen=self.history_len)
        self.text_token = None
        self.text_embedding = None

    # ---- full-window path (reference semantics) -------------------------------------------------------------------------
    def _forward_full(self, image_primary, image_wrist, state, text_token, sample_noise):
        """Full-window mode='test' forward.  With use_cuda_graph the ~2.5 k kernel launches of one action (ViT on 2*S frames,
        resampler, 24-layer backbone, 10 DDIM steps x DiT-B) are captured once and replayed as ONE graph launch."""
        if not self.use_cuda_graph:
            return self.model(image_primary=image_primary, image_wrist=image_wrist, state=state, text_token=text_token,
                              action=None, mode="test", sample_noise=sample_noise)
        if self._graph is None:
            n = self.history_len
            self._static = dict(image_primary=torch.zeros_like(image_primary), image_wrist=torch.zeros_like(image_wrist),
                                state=torch.zeros_like(state), text_token=torch.zeros(1, 77, dtype=text_token.dtype, device=self.device),
                                noise=torch.zeros(n, self.action_pred_steps, 7, device=self.device))
            st = self._static

            def run():
                return self.model(image_primary=st["image_primary"], image_wrist=st["image_wrist"], state=st["state"],
                                  text_token=st["text_token"].unsqueeze(1).expand(1, n, 77), action=None, mode="test",
                                  sample_noise=st["noise"])
            self._graph, self._out = self._capture(run)
        st = self._static
        st["image_primary"].copy_(image_primary)
        st["image_wrist"].copy_(image_wrist)
        st["state"].copy_(state)
        st["text_token"].copy_(text_token[:, 0])
        if sample_noise is None:
            st["noise"].normal_()
        else:
            st["noise"].copy_(sample_noise)
        self._graph.replay()
        return self._out

    @staticmethod
    def _capture(run, warmup=2):
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(warmup):
                run()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = run()
        return g, out

    def window_actions_full(self, sample_noise=None):
        """-> (arm [S, steps, 6], gripper [S, steps, 1]) for every timestep of the padded window + num_step."""
        image_primary = torch.cat(list(self.img_queue), dim=1)
        image_wrist = torch.cat(list(self.gripper_queue), dim=1)
        state = torch.cat(list(self.state_queue), dim=1)
        num_step = image_primary.shape[1]
        if num_step < self.history_len:          # pad with the last frame (:127-131)
            pad = self.history_len - num_step
            image_primary = torch.cat([image_primary, image_primary[:, -1:].expand(-1, pad, -1, -1, -1)], dim=1)
            image_wrist = torch.cat([image_wrist, image_wrist[:, -1:].expand(-1, pad, -1, -1, -1)], dim=1)
            state = torch.cat([state, state[:, -1:].expand(-1, pad, -1)], dim=1)
        out = self._forward_full(image_primary, image_wrist, state, self.text_token, sample_noise)
        return out[0][0], out[1][0], num_step

    # ---- incremental path -------------------------------------------------------------------------------------------------
    def _encode_frame(self, image_primary, image_wrist, state):
        """[1,3,224,224] x2 + [1, state_dim] -> [35, D] token block of this frame (graph replay; returns a fresh copy)."""
        m = self.model
        if not self.use_cuda_graph:
            return m.encode_frame_tokens(image_primary, image_wrist, state)[0]
        if self._enc_graph is None:
            self._enc_static = dict(p=torch.zeros_like(image_primary), w=torch.zeros_like(image_wrist), s=torch.zeros_like(state))
            st = self._enc_static
            self._enc_graph, self._enc_out = self._capture(lambda: m.encode_frame_tokens(st["p"], st["w"], st["s"]))
        st = self._enc_static
        st["p"].copy_(image_primary)
        st["w"].copy_(image_wrist)
        st["s"].copy_(state)
        self._enc_graph.replay()
        return self._enc_out[0].clone()

    def _action_incremental(self, sel, sample_noise):
        m = self.model
        S = self.history_len
        toks = list(self.tok_queue)
        toks = toks + [toks[-1]] * (S - len(toks))                   # padded repeats of the last frame (:127-131)
        frame_tokens = torch.stack(toks, dim=0)
        if not self.use_cuda_graph:
            return m.rollout_action(self.text_embedding, frame_tokens, sel, sample_noise=sample_noise, prune=self.prune)
        if sel not in self._act_graphs:
            st = dict(tok=torch.zeros_like(frame_tokens), txt=torch.zeros_like(self.text_embedding),
                      noise=torch.zeros(1, self.action_pred_steps, 7, device=self.device))
            st["tok"].copy_(frame_tokens)
            st["txt"].copy_(self.text_embedding)
            g, out = self._capture(lambda: m.rollout_action(st["txt"], st["tok"], sel, sample_noise=st["noise"], prune=self.prune))
            self._act_graphs[sel] = (g, st, out)
        g, st, out = self._act_graphs[sel]
        st["tok"].copy_(frame_tokens)
        st["txt"].copy_(self.text_embedding)
        if sample_noise is None:
            st["noise"].normal_()
        else:
            st["noise"].copy_(sample_noise)
        g.replay()
        return out

    # ---- one env step -----------------------------------------------------------------------------------------------------
    def _frame(self, image, flip_vertical=False):
        """-> [1, 1, 3, 224, 224] in the cast dtype on the device.  A raw uint8 [h, w, 3] frame (numpy array or tensor, as the
        simulator returns it) is uploaded as bytes and put through CLIP's image transform on the device (`preprocess_image`,
        the reference's `image_process_fn`, :82-90); a preprocessed [3, 224, 224] tensor is only moved and cast.  A stack of
        n frames ([n, h, w, 3] / [n, 3, 224, 224]) gives [n, 1, 3, 224, 224] the same way, in one call."""
        if isinstance(image, np.ndarray):
            image = torch.from_numpy(np.ascontiguousarray(image))
        if image.dtype != torch.uint8:
            return image.to(self.device, self.cast_type).view(-1, 1, 3, 224, 224)
        out_dtype = self.cast_type if self.cast_type in (torch.float32, torch.bfloat16) else torch.float32
        x = preprocess_image(image.to(self.device), out_dtype, flip_vertical)
        return x.to(self.cast_type).view(-1, 1, 3, 224, 224)

    @torch.no_grad()
    def infer(self, image_static, image_gripper, state_vec, text_tokens, sample_noise=None, flip_static=False):
        """Push one observation, return (arm [steps, 6], gripper [steps, 1], num_step) of the SELECTED timestep.
        image_*: preprocessed [3, 224, 224] tensors or raw uint8 [h, w, 3] frames (see `_frame`; `flip_static` flips a raw
        static frame upside down first).  sample_noise: the DDIM start noise -- [S, steps, 7] (the full-window draw of the
        reference, :944) or [1, steps, 7] (the selected row only)."""
        dev = self.device
        img = self._frame(image_static, flip_static)
        grip = self._frame(image_gripper)
        st = state_vec.to(dev, self.cast_type).view(1, 1, -1)
        assert st.shape[-1] == self.state_dim, f"state has {st.shape[-1]} dims, the model expects {self.state_dim}"
        if self.text_token is None:                              # frozen for the episode (:110-113)
            self.text_token = text_tokens.to(dev).view(1, 1, 77).expand(1, self.history_len, 77)
            if self.incremental:
                self.text_embedding = self.model.encode_text_embedding(text_tokens.to(dev).view(1, 77))
        num_step = min(len(self.tok_queue if self.incremental else self.img_queue) + 1, self.history_len)
        sel = num_step - 1                                       # == -1 once the window is full (:142-145)
        if self.incremental:
            self.tok_queue.append(self._encode_frame(img[:, 0], grip[:, 0], st[:, 0]))
            if sample_noise is not None and sample_noise.shape[0] != 1:
                sample_noise = sample_noise[sel:sel + 1]
            arm, gripper = self._action_incremental(sel, sample_noise)
            return arm[0], gripper[0], num_step
        self.img_queue.append(img)
        self.gripper_queue.append(grip)
        self.state_queue.append(st)
        arm, gripper, _ = self.window_actions_full(sample_noise)
        return arm[sel], gripper[sel], num_step


class ModelWrapper(RolloutEngine):
    """CALVIN rollout wrapper (reference utils/eval_utils_calvin.py:48-147)."""

    def __init__(self, model, cast_dtype=torch.bfloat16, history_len=10, action_pred_steps=3, device="cuda",
                 use_cuda_graph=True, incremental=False, prune=True):
        super().__init__(model, cast_dtype, history_len, action_pred_steps, device, use_cuda_graph, incremental, prune,
                         state_dim=7)

    def reset(self):
        self.reset_window()

    @torch.no_grad()
    def step(self, image_static, image_gripper, robot_obs, text_tokens, sample_noise=None):
        """image_* raw uint8 [h, w, 3] frames (`obs["rgb_obs"]["rgb_static" / "rgb_gripper"]`) or [3,224,224] preprocessed,
        robot_obs [15], text_tokens int [77] -> action [7] (fp16 numpy like the reference)."""
        st = robot_obs.reshape(-1)
        st = torch.cat([st[:6], st[-1:]], dim=-1)                          # :104
        arm, gripper, _ = self.infer(image_static, image_gripper, st, text_tokens, sample_noise)
        action = torch.cat((arm[0].float(), (gripper[0] > 0.5).float()), dim=-1)    # first of the predicted steps (:138)
        action[-1] = (action[-1] - 0.5) * 2                                # scale to -1 or 1 (:139)
        return action.to(torch.float16).cpu().numpy()


class BatchedRolloutEngine(RolloutEngine):
    """`num_envs` rollouts served by one model: one step call takes the observations of any subset of the envs and runs one
    batched encode + one batched action inference for all of them, instead of one `RolloutEngine.infer` per env.

    Per env the window semantics are RolloutEngine's: growing then sliding window of `history_len`, padded by repeating the
    last frame, instruction frozen at the episode's first step, `reset(env)`.  The windows live on the device in window
    order, for all envs at once: the frame-token windows [N, S, 35, D] (incremental=True, `DreamVLA.rollout_actions`, where
    each env selects its timestep on the device) or the preprocessed frames [N, S, 3, 224, 224] x 2 and states
    (incremental=False: a batch-N full-window `mode='test'` forward, the selected row taken per env).  With use_cuda_graph,
    each of these runs as one CUDA graph over all N envs, replayed whatever the envs' fill levels; envs outside the step
    are computed and discarded."""

    def __init__(self, model, num_envs, cast_dtype=torch.bfloat16, history_len=10, action_pred_steps=3, device="cuda",
                 use_cuda_graph=True, incremental=True, state_dim=7):
        self.num_envs = num_envs
        super().__init__(model, cast_dtype, history_len, action_pred_steps, device, use_cuda_graph, incremental, True, state_dim)
        self.fill = [0] * num_envs               # frames pushed since the env's last reset (capped at history_len)
        self.text_set = [False] * num_envs
        self._win = None

    def reset_window(self, env=None):
        if env is None:
            super().reset_window()
            return
        self.fill[env] = 0
        self.text_set[env] = False

    def _alloc(self, tok_shape, text_dtype):
        N, S, dev = self.num_envs, self.history_len, self.device
        steps = self.action_pred_steps
        w = dict(sel=torch.zeros(N, dtype=torch.int32, device=dev), text_token=torch.zeros(N, 77, dtype=text_dtype, device=dev))
        if self.incremental:
            w.update(tok=torch.zeros(N, S, *tok_shape, dtype=self.cast_type, device=dev),
                     txt=torch.zeros(N, tok_shape[-1], dtype=self.cast_type, device=dev),
                     p=torch.zeros(N, 3, 224, 224, dtype=self.cast_type, device=dev),
                     w=torch.zeros(N, 3, 224, 224, dtype=self.cast_type, device=dev),
                     s=torch.zeros(N, self.state_dim, dtype=self.cast_type, device=dev),
                     noise=torch.zeros(N, steps, 7, device=dev))
        else:
            w.update(img=torch.zeros(N, S, 3, 224, 224, dtype=self.cast_type, device=dev),
                     grip=torch.zeros(N, S, 3, 224, 224, dtype=self.cast_type, device=dev),
                     state=torch.zeros(N, S, self.state_dim, dtype=self.cast_type, device=dev),
                     noise=torch.zeros(N * S, steps, 7, device=dev))
        self._win = w

    @staticmethod
    def _push(win, env, n_prev, x):
        """Append x to the window row win[env] that holds n_prev frames: fill (and pad with x) while growing, slide when full."""
        S = win.shape[1]
        if n_prev < S:
            win[env, n_prev:] = x
        else:
            win[env, :-1] = win[env, 1:].clone()
            win[env, -1] = x

    def _encode_frames(self):
        st = self._win
        run = lambda: self.model.encode_frame_tokens(st["p"], st["w"], st["s"])        # noqa: E731
        if not self.use_cuda_graph:
            return run()
        if self._enc_graph is None:
            self._enc_graph, self._enc_out = self._capture(run)
        self._enc_graph.replay()
        return self._enc_out

    def _run_actions(self):
        st = self._win
        N, S = self.num_envs, self.history_len
        if self.incremental:
            def run():
                return self.model.rollout_actions(st["txt"], st["tok"], st["sel"], sample_noise=st["noise"])
        else:
            def run():
                out = self.model(image_primary=st["img"], image_wrist=st["grip"], state=st["state"],
                                 text_token=st["text_token"].unsqueeze(1).expand(N, S, 77), action=None, mode="test",
                                 sample_noise=st["noise"])
                rows = torch.arange(N, device=st["sel"].device) * S + st["sel"].long()
                return out[0][0].index_select(0, rows), out[1][0].index_select(0, rows)
        if not self.use_cuda_graph:
            return run()
        if self._graph is None:
            self._graph, self._out = self._capture(run)
        self._graph.replay()
        return self._out

    @torch.no_grad()
    def infer_batch(self, envs, image_static, image_gripper, states, text_tokens, sample_noise=None, flip_static=False):
        """One observation for each env in `envs` (distinct indices < num_envs) -> (arm [n, steps, 6], gripper [n, steps, 1],
        num_step list) of each env's selected timestep.
        image_*: stacked [n, h, w, 3] uint8 frames (or a list of them, preprocessed on the device in one call) or preprocessed
        [n, 3, 224, 224]; states [n, state_dim]; text_tokens int [n, 77] (read at an env's first step after a reset only).
        sample_noise: [n, steps, 7] start noise of the selected rows, or None (drawn on the device)."""
        envs = [int(e) for e in envs]
        n, S, dev = len(envs), self.history_len, self.device
        assert n and len(set(envs)) == n and all(0 <= e < self.num_envs for e in envs), envs

        def stack(x):
            if isinstance(x, (list, tuple)):
                x = [torch.from_numpy(np.ascontiguousarray(f)) if isinstance(f, np.ndarray) else f for f in x]
                x = torch.stack(x)
            return torch.from_numpy(np.ascontiguousarray(x)) if isinstance(x, np.ndarray) else x
        img = self._frame(stack(image_static), flip_static)[:, 0]                          # [n, 3, 224, 224]
        grip = self._frame(stack(image_gripper))[:, 0]
        st = torch.as_tensor(stack(states)).to(dev, self.cast_type).view(n, -1)
        assert st.shape[-1] == self.state_dim, f"state has {st.shape[-1]} dims, the model expects {self.state_dim}"
        text_tokens = torch.as_tensor(stack(text_tokens)).to(dev).view(n, 77)
        if self._win is None:
            tok_shape = None
            if self.incremental:
                tok_shape = self.model.encode_frame_tokens(img[:1], grip[:1], st[:1]).shape[1:]
            self._alloc(tok_shape, text_tokens.dtype)
        w = self._win
        idx = torch.tensor(envs, device=dev)
        new = [i for i, e in enumerate(envs) if not self.text_set[e]]
        if new:                                                  # frozen for the episode (:110-113)
            rows = torch.tensor(new, device=dev)
            w["text_token"].index_copy_(0, idx[rows], text_tokens[rows])
            if self.incremental:
                w["txt"].index_copy_(0, idx[rows], self.model.encode_text_embedding(text_tokens[rows]).to(self.cast_type))
            for i in new:
                self.text_set[envs[i]] = True
        if self.incremental:
            w["p"].index_copy_(0, idx, img)
            w["w"].index_copy_(0, idx, grip)
            w["s"].index_copy_(0, idx, st)
            toks = self._encode_frames().index_select(0, idx)
        num_steps = []
        for i, e in enumerate(envs):
            if self.incremental:
                self._push(w["tok"], e, self.fill[e], toks[i])
            else:
                self._push(w["img"], e, self.fill[e], img[i])
                self._push(w["grip"], e, self.fill[e], grip[i])
                self._push(w["state"], e, self.fill[e], st[i])
            self.fill[e] = min(self.fill[e] + 1, S)
            num_steps.append(self.fill[e])
        sel = torch.tensor([max(f - 1, 0) for f in self.fill], dtype=torch.int32)    # == -1 once full (:142-145)
        w["sel"].copy_(sel)
        if sample_noise is None:
            w["noise"].normal_()
        elif self.incremental:
            w["noise"].index_copy_(0, idx, sample_noise.to(dev, torch.float32))
        else:                                                    # the selected row of each env's [S, steps, 7] draw
            w["noise"].view(self.num_envs, S, *w["noise"].shape[1:])[idx, sel.to(dev).long()[idx]] = \
                sample_noise.to(dev, torch.float32)
        arm, gripper = self._run_actions()
        return arm.index_select(0, idx), gripper.index_select(0, idx), num_steps


class BatchedModelWrapper(BatchedRolloutEngine):
    """CALVIN rollout wrapper for `num_envs` environments: `ModelWrapper.step` per env, batched (see BatchedRolloutEngine)."""

    def __init__(self, model, num_envs, cast_dtype=torch.bfloat16, history_len=10, action_pred_steps=3, device="cuda",
                 use_cuda_graph=True, incremental=True):
        super().__init__(model, num_envs, cast_dtype, history_len, action_pred_steps, device, use_cuda_graph, incremental,
                         state_dim=7)

    def reset(self, env):
        self.reset_window(env)

    @torch.no_grad()
    def step(self, envs, image_static, image_gripper, robot_obs, text_tokens, sample_noise=None):
        """robot_obs [n, 15], text_tokens int [n, 77], images as `infer_batch` takes them -> actions [n, 7] (fp16 numpy)."""
        obs = torch.as_tensor(np.asarray(robot_obs) if not torch.is_tensor(robot_obs) else robot_obs).reshape(len(envs), -1)
        st = torch.cat([obs[:, :6], obs[:, -1:]], dim=-1)                  # :104
        arm, gripper, _ = self.infer_batch(envs, image_static, image_gripper, st, text_tokens, sample_noise)
        action = torch.cat((arm[:, 0].float(), (gripper[:, 0] > 0.5).float()), dim=-1)   # first of the predicted steps (:138)
        action[:, -1] = (action[:, -1] - 0.5) * 2                          # scale to -1 or 1 (:139)
        return action.to(torch.float16).cpu().numpy()
