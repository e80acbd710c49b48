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
        the reference's `image_process_fn`, :82-90); a preprocessed [3, 224, 224] tensor is only moved and cast."""
        if isinstance(image, np.ndarray):
            image = torch.from_numpy(np.ascontiguousarray(image))
        if image.dtype != torch.uint8:
            return image.to(self.device, self.cast_type).view(1, 1, 3, 224, 224)
        out_dtype = self.cast_type if self.cast_type in (torch.float32, torch.bfloat16) else torch.float32
        x = preprocess_image(image.to(self.device), out_dtype, flip_vertical)
        return x.to(self.cast_type).view(1, 1, 3, 224, 224)

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
