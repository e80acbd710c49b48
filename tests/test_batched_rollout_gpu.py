"""Batched rollouts on the GPU: the attention forward under a per-sequence mask stack against one call per mask and an fp32
softmax; DreamVLA.rollout_actions against per-env rollout_action(prune=True); the batched CALVIN / LIBERO wrappers against
one single-env wrapper per env, with staggered resets and envs left out of steps."""
import ctypes

import numpy as np
import pytest
import torch

from tests import synth
from tests.test_rollout_gpu import build, observations

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


@pytest.mark.parametrize("L", [80, 200])          # Lq < 96: mma.sync kernel; >= 96: wgmma kernel
def test_attention_mask_index_equals_per_mask_calls(dev, L):
    from dreamvla_b200 import ops
    B, H, n = 5, 3, 3
    g = torch.Generator().manual_seed(L)
    qkv = (torch.randn(B, L, 3, H, 64, generator=g)).to(dev, torch.bfloat16)
    vis = torch.rand(n, L, L, generator=g) < 0.4
    vis |= torch.eye(L, dtype=torch.bool)                                   # every row sees at least itself
    vis[1, :, :L // 2] = False                                              # whole tiles skipped in one mask
    vis[1] |= torch.eye(L, dtype=torch.bool)
    vis[2] = torch.ones(L, L, dtype=torch.bool).tril()
    index = torch.tensor([2, 0, 1, 2, 1], dtype=torch.int32, device=dev)
    stack = ops.AttnMaskStack(vis, dev)
    with torch.no_grad():
        got = ops.self_attention_fused(qkv, 0.125, stack.select(index))
        for b in range(B):
            want = ops.self_attention_fused(qkv[b:b + 1].contiguous(), 0.125, ops.AttnMask(vis[int(index[b])], dev))
            assert torch.equal(got[b:b + 1], want), b
    q, k, v = (qkv[:, :, i].float().permute(0, 2, 1, 3) for i in range(3))
    s = (q @ k.transpose(-1, -2)) * 0.125
    s = s.masked_fill(~vis[index.long().cpu()].to(dev).unsqueeze(1), float("-inf"))
    ref = (s.softmax(-1) @ v).permute(0, 2, 1, 3)
    err = float((got.float() - ref).norm() / ref.norm())
    assert err < 1e-2, err
    with pytest.raises(RuntimeError, match="forward only"):
        ops.self_attention_fused(qkv.clone().requires_grad_(True), 0.125, stack.select(index))


def gemm_plan(M, N, K):
    from dreamvla_b200 import _lib
    a = _lib.GemmArgs()
    a.a, a.b, a.out = 1 << 40, 2 << 40, 3 << 40                  # planning only: never dereferenced
    a.M, a.N, a.K, a.lda, a.ldb, a.ldo, a.alpha = M, N, K, K, N, N, 1.0
    a.b_mn_major = 1                                              # HF Conv1D weight [in, out]
    a.workspace, a.workspace_bytes = 4 << 40, int(_lib.load().dvla_gemm_workspace_bytes(None))
    info = _lib.GemmPlanInfo()
    assert _lib.load().dvla_gemm_plan(ctypes.byref(a), ctypes.byref(info)) == 0, _lib.load().dvla_last_error()
    return info


def batch_invariant(m_single, m_batched, N, K):
    """True when dvla_gemm runs both row counts on the same kernel with every output tile one CTA's whole-K sum in a fixed
    order (no split-K, no K-split tail): then a row's values do not depend on how many other rows share the call."""
    a, b = gemm_plan(m_single, N, K), gemm_plan(m_batched, N, K)
    return a.kernel == b.kernel and all(p.tail_splits <= 1 and p.k_splits <= 1 for p in (a, b))


def window(model, S, dev, seed):
    g = torch.Generator().manual_seed(seed)
    text = torch.zeros(77, dtype=torch.long)
    text[0], text[1:6], text[6] = 49406, torch.randint(1, 49406, (5,), generator=g), 49407
    img, grip = torch.randn(S, 3, 224, 224, generator=g), torch.randn(S, 3, 224, 224, generator=g)
    st = torch.randn(S, 8 if model.gripper_width else 7, generator=g) * 0.5
    with torch.no_grad():
        toks = model.encode_frame_tokens(img.to(dev, torch.bfloat16), grip.to(dev, torch.bfloat16), st.to(dev, torch.bfloat16))
        txt = model.encode_text_embedding(text.to(dev).view(1, 77))
    return txt, toks


@pytest.mark.parametrize("case", ["libero_dit", "calvin_allheads"])
def test_rollout_actions_equals_per_env_rollout_action(dev, case):
    """Each env's sequence is its pruned single-env sequence followed by A slots no kept row sees, and the backbone's GEMMs
    sum every output tile over the whole K in one order at both row counts (asserted through dvla_gemm_plan), so every kept
    row is computed as in the single-env call."""
    cfg = synth.CASES[case]
    S, D = cfg["sequence_length"], cfg["hidden_dim"]
    model = build(cfg, dev)
    model.FUSED_SAMPLER = False
    N = 4
    sels = [(e * 2 + 1) % S for e in range(N)]
    wins = [window(model, S, dev, 100 + e) for e in range(N)]
    txt = torch.cat([w[0] for w in wins])
    toks = torch.stack([w[1] for w in wins])
    sel = torch.tensor(sels, dtype=torch.int32, device=dev)
    Lb = model._batched_rollout_tables(dev)[1].shape[1]
    for s_ in sels:
        m_single = len(model._rollout_mask(s_, True, dev)[2])
        for n_out, k in ((3 * D, D), (D, D), (4 * D, D), (D, 4 * D)):       # c_attn, c_proj, c_fc, mlp c_proj
            assert batch_invariant(m_single, N * Lb, n_out, k), (case, s_, n_out, k)
    noise = torch.randn(N, 3, 7, generator=torch.Generator().manual_seed(3)).to(dev)
    with torch.no_grad():
        feat = model.rollout_actions(txt, toks, sel, return_features=True)
        arm, grip = model.rollout_actions(txt, toks, sel, sample_noise=noise)
        for e in range(N):
            f1 = model.rollout_action(txt[e:e + 1], toks[e], sels[e], prune=True, return_features=True)
            a1, g1 = model.rollout_action(txt[e:e + 1], toks[e], sels[e], sample_noise=noise[e:e + 1], prune=True)
            assert torch.equal(feat[e:e + 1], f1), (case, e, float((feat[e:e + 1].float() - f1.float()).abs().max()))
            assert torch.equal(arm[e:e + 1], a1) and torch.equal(grip[e:e + 1], g1), (case, e)


def test_batched_calvin_wrapper_matches_single_env_wrappers(dev):
    from dreamvla_b200.utils.eval_utils_calvin import BatchedModelWrapper, ModelWrapper
    cfg = synth.CASES["libero_dit"]
    S = cfg["sequence_length"]
    model = build(cfg, dev)
    model.FUSED_SAMPLER = False
    N, T = 3, 2 * S + 3
    streams = [observations(T, seed=40 + e) for e in range(N)]
    singles = [ModelWrapper(model, history_len=S, device=dev, use_cuda_graph=False, incremental=True, prune=True)
               for _ in range(N)]
    batched = BatchedModelWrapper(model, N, history_len=S, device=dev, use_cuda_graph=True)
    eager = BatchedModelWrapper(model, N, history_len=S, device=dev, use_cuda_graph=False)
    g = torch.Generator().manual_seed(8)
    pos = [0] * N
    for t in range(T):
        envs = [e for e in range(N) if (t + e) % 4 != 3]                  # one env sits a step out now and then
        for e in envs:
            if t == 2 * e + 1 or (e == 0 and t == S + 1):                  # staggered episode starts
                singles[e].reset()
                batched.reset(e)
                eager.reset(e)
        noise = torch.randn(len(envs), 3, 7, generator=g)
        ims = torch.stack([streams[e][1][pos[e]][0] for e in envs])
        grs = torch.stack([streams[e][1][pos[e]][1] for e in envs])
        obs = torch.stack([streams[e][1][pos[e]][2] for e in envs])
        txt = torch.stack([streams[e][0] if t < S else streams[(e + 1) % N][0] for e in envs])   # later texts are ignored
        got = batched.step(envs, ims, grs, obs, txt, sample_noise=noise)
        ref_eager = eager.step(envs, ims, grs, obs, txt, sample_noise=noise)
        assert np.array_equal(got, ref_eager), t
        for i, e in enumerate(envs):
            want = singles[e].step(ims[i], grs[i], obs[i], txt[i], sample_noise=noise[i:i + 1])
            assert batched.fill[e] == len(singles[e].tok_queue), (t, e)
            assert np.array_equal(got[i], want), (t, e, got[i], want)
            pos[e] += 1


@pytest.mark.parametrize("ensembling", [False, True])
def test_batched_libero_wrapper_matches_single_env_wrappers(dev, ensembling):
    from dreamvla_b200.utils.eval_utils_libero import BatchedModelWrapper, ModelWrapper
    cfg = synth.CPU_ONLY_CASES["libero_gripper_width"]
    S = cfg["sequence_length"]
    model = build(cfg, dev)
    model.FUSED_SAMPLER = False
    N, T = 3, S + 3
    kw = dict(history_len=S, use_ensembling=ensembling, libero_eval_max_steps=16, gripper_width=True, device=dev)
    singles = [ModelWrapper(model, use_cuda_graph=False, incremental=True, prune=True, **kw) for _ in range(N)]
    batched = BatchedModelWrapper(model, N, use_cuda_graph=True, **kw)
    g = torch.Generator().manual_seed(21)
    text, _ = observations(1, seed=3)
    ts = [0] * N
    for e in range(N):
        singles[e].reset()
        batched.reset(e)
    for t in range(T):
        envs = [e for e in range(N) if t >= e]                              # envs join one step apart
        n = len(envs)
        img = torch.randint(0, 256, (n, 96, 128, 3), dtype=torch.uint8, generator=g)   # raw frames: flip + preprocessing
        grip = torch.randint(0, 256, (n, 96, 128, 3), dtype=torch.uint8, generator=g)
        pos, quat = torch.randn(n, 3, generator=g).numpy() * 0.3, torch.randn(n, 4, generator=g).numpy()
        qpos = torch.rand(n, 2, generator=g).numpy() * 0.04
        noise = torch.randn(n, 3, 7, generator=g)
        got = batched.step(envs, img, grip, pos, quat, qpos, text.expand(n, 77), [ts[e] for e in envs], sample_noise=noise)
        for i, e in enumerate(envs):
            want = singles[e].step(img[i].numpy(), grip[i].numpy(), pos[i], quat[i], qpos[i], text, ts[e],
                                   sample_noise=noise[i:i + 1])
            assert np.array_equal(np.asarray(got[i], dtype=np.float64), np.asarray(want, dtype=np.float64)), (t, e, got[i], want)
            ts[e] += 1


def test_batched_full_window_wrapper_matches_single_env_wrappers(dev):
    """incremental=False: a batch-N mode='test' forward over the device windows with each env's row picked, against one
    full-window ModelWrapper per env fed the same observations, resets and noise (the selected row's noise in the batched
    call, that row of an [S, steps, 7] draw in the single one).  Window bookkeeping is exact; the actions agree to the
    rounding of a batch-N forward against batch-1 ones (the ViT's GEMMs at N·2S frames may cut other K ranges), under the
    bar of test_incremental_rollout_matches_full_window; graph and eager batched runs are bit-identical."""
    from dreamvla_b200.utils.eval_utils_calvin import BatchedModelWrapper, ModelWrapper
    cfg = synth.CASES["libero_dit"]
    S = cfg["sequence_length"]
    model = build(cfg, dev)
    N, T = 3, 2 * S + 2
    streams = [observations(T, seed=60 + e) for e in range(N)]
    singles = [ModelWrapper(model, history_len=S, device=dev, use_cuda_graph=False) for _ in range(N)]
    batched = BatchedModelWrapper(model, N, history_len=S, device=dev, use_cuda_graph=True, incremental=False)
    eager = BatchedModelWrapper(model, N, history_len=S, device=dev, use_cuda_graph=False, incremental=False)
    g = torch.Generator().manual_seed(12)
    pos = [0] * N
    worst = 0.0
    for t in range(T):
        envs = [e for e in range(N) if (t + e) % 4 != 3]
        for e in envs:
            if t == 2 * e + 1:
                singles[e].reset()
                batched.reset(e)
                eager.reset(e)
        full = torch.randn(len(envs), S, 3, 7, generator=g)
        sel = [min(batched.fill[e] + 1, S) - 1 for e in envs]
        noise = torch.stack([full[i, s] for i, s in enumerate(sel)])
        ims = torch.stack([streams[e][1][pos[e]][0] for e in envs])
        grs = torch.stack([streams[e][1][pos[e]][1] for e in envs])
        obs = torch.stack([streams[e][1][pos[e]][2] for e in envs])
        txt = torch.stack([streams[e][0] for e in envs])
        got = batched.step(envs, ims, grs, obs, txt, sample_noise=noise)
        assert np.array_equal(got, eager.step(envs, ims, grs, obs, txt, sample_noise=noise)), t
        for i, e in enumerate(envs):
            want = singles[e].step(ims[i], grs[i], obs[i], txt[i], sample_noise=full[i])
            assert batched.fill[e] == len(singles[e].img_queue), (t, e)
            a, b = got[i].astype(np.float32), want.astype(np.float32)
            err = float(np.abs(a[:6] - b[:6]).max() / (np.abs(b[:6]).max() + 1e-6))
            worst = max(worst, err)
            assert err < 0.3, (t, e, a, b)
            pos[e] += 1
    print(f"batched full window vs single-env wrappers: worst relative action difference {worst:.3e}")
