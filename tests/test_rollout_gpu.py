"""Rollout wrappers on the GPU: window / padding / row-selection semantics of `ModelWrapper.step`
(reference utils/eval_utils_calvin.py:107-145, utils/eval_utils_libero.py:94-179) against direct `mode='test'` forwards,
and rollout-level incremental inference (SURVEY §8 f-1) against the full-window path."""
import numpy as np
import pytest
import torch

from tests import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def build(cfg, dev):
    from dreamvla_b200.models import DreamVLA
    torch.manual_seed(0)
    m = DreamVLA(finetune_type="calvin", clip_device="cpu", vit_checkpoint_path=None, **synth.ctor_kwargs(cfg))
    m.load_state_dict(synth.synth_state_dict(m.state_dict(), cfg["weight_seed"]))
    m = m.bfloat16().to(dev)
    m._init_model_type()
    return m.eval()


def observations(n, seed, state_dim=15):
    g = torch.Generator().manual_seed(seed)
    text = torch.zeros(77, dtype=torch.long)
    text[0], text[1:6], text[6] = 49406, torch.randint(1, 49406, (5,), generator=g), 49407
    obs = [(torch.randn(3, 224, 224, generator=g), torch.randn(3, 224, 224, generator=g), torch.randn(state_dim, generator=g) * 0.5)
           for _ in range(n)]
    return text, obs


def reference_window_action(model, history, text, noise, S, dev):
    """The reference's step, spelled out (eval_utils_calvin.py:107-145): window of the last S observations, padded by
    repeating the last one, full mode='test' forward, first predicted step of row num_step-1 (or the last row)."""
    frames = history[-S:]
    num_step = len(frames)
    frames = frames + [frames[-1]] * (S - num_step)
    ip = torch.stack([f[0] for f in frames]).unsqueeze(0).to(dev, torch.bfloat16)
    iw = torch.stack([f[1] for f in frames]).unsqueeze(0).to(dev, torch.bfloat16)
    st = torch.stack([torch.cat([f[2][:6], f[2][-1:]]) for f in frames]).unsqueeze(0).to(dev, torch.bfloat16)
    tt = text.to(dev).view(1, 1, 77).repeat(1, S, 1)
    with torch.no_grad():
        out = model(image_primary=ip, image_wrist=iw, state=st, text_token=tt, action=None, mode="test", sample_noise=noise.to(dev))
    arm, grip = out[0], out[1]
    action = torch.concat((arm[0, :, 0, :], grip[0, :, 0, :] > 0.5), dim=-1)
    action[:, -1] = (action[:, -1] - 0.5) * 2
    action = action.cpu().detach().to(dtype=torch.float16).numpy()
    return action[num_step - 1] if num_step < S else action[-1]


@pytest.mark.parametrize("graph", [False, True])
def test_modelwrapper_step_window_semantics(dev, graph):
    from dreamvla_b200.utils.eval_utils_calvin import ModelWrapper
    cfg = synth.CASES["libero_dit"]                       # 2 layers, S = 3, DiT head
    S = cfg["sequence_length"]
    model = build(cfg, dev)
    text, obs = observations(S + 3, seed=5)
    w = ModelWrapper(model, history_len=S, action_pred_steps=3, device=dev, use_cuda_graph=graph)
    g = torch.Generator().manual_seed(9)
    for i in range(len(obs)):                             # growing window (1..S), then sliding
        noise = torch.randn(S, 3, 7, generator=g)
        got = w.step(*obs[i], text, sample_noise=noise)
        want = reference_window_action(model, obs[:i + 1], text, noise, S, dev)
        assert got.dtype == np.float16 and got.shape == (7,)
        assert np.array_equal(got, want), (i, got, want)
    # a changed instruction mid-episode is ignored until reset() (:110-113)
    other = text.clone()
    other[1:6] = (other[1:6] + 17) % 49000 + 1
    noise = torch.randn(S, 3, 7, generator=g)
    a = w.step(*obs[-1], other, sample_noise=noise)
    b = reference_window_action(model, obs + [obs[-1]], text, noise, S, dev)
    assert np.array_equal(a, b)
    w.reset()
    assert len(w.img_queue) == 0 and w.text_token is None


@pytest.mark.parametrize("case,prune", [("libero_dit", False), ("libero_dit", True), ("calvin_allheads", True)])
def test_incremental_rollout_matches_full_window(dev, case, prune):
    """Per-frame token cache + selected-timestep-only backbone rows / DDIM vs the full-window forward, both through CUDA
    graphs and with wrappers of both kinds alive on the same model (they share its lazily built tables).
    prune=False feeds the backbone the same L tokens as the full window: the selected rows see identical inputs, so the
    actions agree to the last bit of the fp16 action the wrapper returns.
    prune=True drops never-attended tokens: the same mathematics on another sequence length, i.e. other flash-attention
    tiles.  The backbone's action-token rows
    -- the quantity the pruning touches -- agree to bf16 rounding; the 10-step guided sampler on top of random synthetic
    weights amplifies that, so the actions get a wide bar (a trained model's sampler is far better conditioned)."""
    from dreamvla_b200.utils.eval_utils_calvin import ModelWrapper
    cfg = synth.CASES[case]
    S = cfg["sequence_length"]
    model = build(cfg, dev)
    model.FUSED_SAMPLER = False          # same sampler code on both sides: this test is about the token cache / row pruning
    text, obs = observations(S + 3, seed=11)
    full = ModelWrapper(model, history_len=S, device=dev, use_cuda_graph=True)
    inc = ModelWrapper(model, history_len=S, device=dev, use_cuda_graph=True, incremental=True, prune=prune)
    g = torch.Generator().manual_seed(4)
    worst = worst_feat = 0.0
    for i in range(len(obs)):
        noise = torch.randn(S, 3, 7, generator=g)
        a = full.step(*obs[i], text, sample_noise=noise).astype(np.float32)
        b = inc.step(*obs[i], text, sample_noise=noise).astype(np.float32)
        assert np.isfinite(b).all(), (i, b)
        err = float(np.abs(a[:6] - b[:6]).max() / (np.abs(a[:6]).max() + 1e-6))
        worst = max(worst, err)
        if not prune:
            assert np.array_equal(a, b), (i, a, b)
            continue
        assert err < 0.3, (i, a, b)
        toks = list(inc.tok_queue)
        frames = torch.stack(toks + [toks[-1]] * (S - len(toks)))
        sel = min(i, S - 1)
        f0 = model.rollout_action(inc.text_embedding, frames, sel, prune=False, return_features=True).float()
        f1 = model.rollout_action(inc.text_embedding, frames, sel, prune=True, return_features=True).float()
        e = float((f0 - f1).norm() / f0.norm())
        worst_feat = max(worst_feat, e)
        assert e < 1e-2, (i, e)
    print(f"incremental[{case}, prune={prune}] worst relative action difference {worst:.3e}; backbone action rows rel-L2 {worst_feat:.3e}")


def test_fused_sampler_matches_module_sampler_and_oracle(dev):
    """csrc/dit_sampler.cu (one persistent kernel for the whole guided DDIM loop) against the module path (DiT blocks on the
    GEMM / attention kernels + torch DDIM algebra) and against the fp32 oracle (oracle.Diffusion.ddim_loop + dit_forward,
    pinned to the reference by the test-mode goldens)."""
    from oracle import dreamvla_oracle as O
    cfg = synth.CASES["libero_dit"]
    model = build(cfg, dev)
    sd = {k: v.detach().float().cpu() for k, v in model.state_dict().items() if k.startswith("action_model.")}
    g = torch.Generator().manual_seed(17)
    worst = []
    for bs in (1,):                     # the fused kernel is the one-sequence (rollout) case
        feat = (torch.randn(bs, 3, 1024, generator=g) * 0.7).to(torch.bfloat16)
        noise = torch.randn(bs, 3, 7, generator=g)
        with torch.no_grad():
            model.FUSED_SAMPLER = True
            a = model._ddim_actions(feat.to(dev), noise.to(dev), dev).float().cpu()
            model.FUSED_SAMPLER = False
            b = model._ddim_actions(feat.to(dev), noise.to(dev), dev).float().cpu()
            # oracle: same guidance construction as dreamvla_model.py:944-987
            unc = sd["action_model.net.z_embedder.uncondition"].unsqueeze(0).expand(bs, 3, -1)
            z = torch.cat([feat.float(), unc], 0)
            x0 = torch.cat([noise.to(torch.bfloat16).float()] * 2, 0)

            def cfg_model(x, t):
                half = x[: len(x) // 2]
                out = O.dit_forward(sd, torch.cat([half, half], 0), t, z)
                cond, uncond = torch.split(out, len(out) // 2, dim=0)
                e = uncond + 1.5 * (cond - uncond)
                return torch.cat([e, e], 0)
            ref = O.Diffusion(100, use=set(range(0, 100, 10))).ddim_loop(cfg_model, x0)[:bs]
        e_fused, e_mod = float((a - ref).norm() / ref.norm()), float((b - ref).norm() / ref.norm())
        worst.append((bs, e_fused, e_mod, float((a - b).norm() / b.norm())))
        assert torch.isfinite(a).all()
        assert e_fused <= e_mod + 5e-3, worst
    print("fused sampler: " + "; ".join(f"bs={bs}: vs oracle fused {ef:.3e} / module {em:.3e}, fused vs module {d:.3e}"
                                        for bs, ef, em, d in worst))


@pytest.mark.parametrize("ensembling", [False, True])
def test_libero_wrapper_gripper_width(dev, ensembling):
    """8-dim `--gripper_width` state through the LIBERO wrapper (eval_utils_libero.py:112-115) vs a direct forward; the
    incremental engine under the same wrapper agrees."""
    from dreamvla_b200.utils.eval_utils_libero import ModelWrapper, quaternion_to_euler
    cfg = synth.CPU_ONLY_CASES["libero_gripper_width"]
    S = cfg["sequence_length"]
    model = build(cfg, dev)
    model.FUSED_SAMPLER = False          # the same sampler code in both wrappers: this test compares them bit for bit
    g = torch.Generator().manual_seed(21)
    text, _ = observations(1, seed=3)
    w = ModelWrapper(model, history_len=S, use_ensembling=ensembling, libero_eval_max_steps=16, gripper_width=True, device=dev,
                     use_cuda_graph=False)
    wi = ModelWrapper(model, history_len=S, use_ensembling=ensembling, libero_eval_max_steps=16, gripper_width=True, device=dev,
                      use_cuda_graph=True, incremental=True, prune=False)
    w.reset()
    wi.reset()
    hist = []
    for t in range(S + 2):
        img, grip = torch.randn(3, 224, 224, generator=g), torch.randn(3, 224, 224, generator=g)
        pos, quat, qpos = torch.randn(3, generator=g).numpy() * 0.3, torch.randn(4, generator=g).numpy(), torch.rand(2, generator=g).numpy() * 0.04
        noise = torch.randn(S, 3, 7, generator=g)
        a = w.step(img, grip, pos, quat, qpos, text, t, sample_noise=noise)
        b = wi.step(img, grip, pos, quat, qpos, text, t, sample_noise=noise)
        assert a.shape == (7,) and a[-1] in (-1.0, 1.0)
        assert np.allclose(np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64), atol=0, rtol=0), (t, a, b)
        st = torch.from_numpy(np.concatenate([pos, quaternion_to_euler(quat), qpos]))
        hist.append((img, grip, st))
        if not ensembling:
            frames = hist[-S:]
            n = len(frames)
            frames = frames + [frames[-1]] * (S - n)
            with torch.no_grad():
                out = model(image_primary=torch.stack([f[0] for f in frames]).unsqueeze(0).to(dev, torch.bfloat16),
                            image_wrist=torch.stack([f[1] for f in frames]).unsqueeze(0).to(dev, torch.bfloat16),
                            state=torch.stack([f[2] for f in frames]).unsqueeze(0).to(dev, torch.bfloat16),
                            text_token=text.to(dev).view(1, 1, 77).repeat(1, S, 1), mode="test", sample_noise=noise.to(dev))
            row = n - 1 if n < S else -1
            want = torch.cat((out[0][0, row, 0].float(), (out[1][0, row, 0] > 0.5).float() * 2 - 1)).to(torch.float16).cpu().numpy()
            assert np.array_equal(a, want), (t, a, want)
