"""`--dit_type` DiT-S (head_dim 96) and DiT-L (depth 24, hidden 1024) action heads on the GPU: the head_dim-96 short-sequence
attention kernels against fp32 torch, the model against the reference goldens and the fp32 oracle (forward and gradients),
the fused DDIM sampler against the module path and the oracle, incremental rollouts, and train.py's entry point."""
import json
import os

import numpy as np
import pytest
import torch

from tests import synth
from tests.dit_types import DIT_SIZES, DIT_TYPE_CASES, ctor_kwargs, oracle_forward

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return float((a - b).norm() / (b.norm() + 1e-12))


def build(cfg, dev):
    """The product model of a DIT_TYPE_CASES configuration with its synthetic weights, bf16 on the GPU, dropouts off (as
    test_model_gpu.build, with the action-head size passed on).  Returns (model, fp32 state_dict)."""
    from dreamvla_b200.models import DreamVLA
    torch.manual_seed(0)
    m = DreamVLA(finetune_type="calvin", clip_device="cpu", vit_checkpoint_path=None, **ctor_kwargs(cfg))
    sd = synth.synth_state_dict(m.state_dict(), cfg["weight_seed"])
    m.load_state_dict(sd)
    m = m.bfloat16().to(dev)
    m._init_model_type()
    gp = m.transformer_backbone
    gp.embd_pdrop = 0.0
    for blk in gp.h:
        blk.attn.attn_pdrop = blk.attn.resid_pdrop = blk.mlp.resid_pdrop = 0.0
    return m, sd


# ---- head_dim 96 on the short-sequence kernels (attention_small.cu) -------------------------------------------------------
HD = 96
# (B, H, Lq, Lk): the DiT-S blocks (8*B*S sequences of 6 tokens, 4 heads), a single query, the largest short case, Lq != Lk
ATTN_SHAPES = {"dit": (40, 4, 6, 6), "lq1": (6, 4, 1, 6), "lq32_lk64": (3, 4, 32, 64), "lq_ne_lk": (5, 4, 5, 17)}
ATTN_CASES = [(s, lay, kb) for s in ATTN_SHAPES for lay in ("strided", "fused") for kb in (False, True)
              if lay == "strided" or ATTN_SHAPES[s][2] == ATTN_SHAPES[s][3]]


def _operands(shape, layout, dev, g):
    """q, k, v (bf16) and empty dq, dk, dv in the given layout:
    strided: three separate [B, H, L, 96] tensors viewed as [B, L, H, 96] (head stride L*96, sequence stride 96);
    fused:   slices of one [B, L, 3, H, 96] buffer, the gradients slices of one such buffer (the DiT's own layout)."""
    B, H, Lq, Lk = shape
    if layout == "fused":
        qkv = torch.randn(B, Lq, 3, H, HD, generator=g).to(dev, torch.bfloat16)
        dqkv = torch.empty_like(qkv)
        return [qkv[:, :, i] for i in range(3)], [dqkv[:, :, i] for i in range(3)]
    qkv = [torch.randn(B, H, n, HD, generator=g).to(dev, torch.bfloat16).permute(0, 2, 1, 3) for n in (Lq, Lk, Lk)]
    grads = [torch.empty(B, H, n, HD, device=dev, dtype=torch.bfloat16).permute(0, 2, 1, 3) for n in (Lq, Lk, Lk)]
    return qkv, grads


@pytest.mark.parametrize("shape,layout,key_bias", ATTN_CASES)
def test_hd96_attention_matches_fp32_torch(dev, shape, layout, key_bias):
    from dreamvla_b200 import _lib as L
    g = torch.Generator().manual_seed(ATTN_CASES.index((shape, layout, key_bias)))
    B, H, Lq, Lk = ATTN_SHAPES[shape]
    (q, k, v), (dq, dk, dv) = _operands(ATTN_SHAPES[shape], layout, dev, g)
    # key_bias as the decoders pass it (dreamvla_model.py:803-806): log r for a key that stands for r identical keys
    bias = torch.randint(1, 5, (Lk,), generator=g).float().log().to(dev) if key_bias else None
    scale = HD ** -0.5
    o, lse = L.attn_fwd(q, k, v, scale, key_bias=bias)
    d_o = torch.randn(B, Lq, H, HD, generator=g).to(dev, torch.bfloat16)
    L.attn_bwd(q, k, v, o, d_o, lse, scale, dq, dk, dv, key_bias=bias)
    qf, kf, vf = (t.detach().float().requires_grad_(True) for t in (q, k, v))
    s = torch.einsum("bihd,bjhd->bhij", qf, kf) * scale
    if bias is not None:
        s = s + bias.float()
    oref = torch.einsum("bhij,bjhd->bihd", torch.softmax(s, dim=-1), vf)
    oref.backward(d_o.float())
    errs = {"o": rel(o, oref), "dq": rel(dq, qf.grad), "dk": rel(dk, kf.grad), "dv": rel(dv, vf.grad)}
    lse_err = float((lse - torch.logsumexp(s, dim=-1).detach()).abs().max())
    assert all(e <= 2.5e-3 for e in errs.values()), errs
    assert lse_err <= 2e-5, lse_err


def test_hd96_fused_self_attention_autograd(dev):
    """ops.self_attention_fused at head_dim 96: the backward writes the fused [B, L, 3, H, 96] gradient."""
    from dreamvla_b200 import ops
    g = torch.Generator().manual_seed(5)
    qkv = torch.randn(16, 6, 3, 4, HD, generator=g).to(dev, torch.bfloat16).requires_grad_(True)
    o = ops.self_attention_fused(qkv, HD ** -0.5)
    d_o = torch.randn(o.shape, generator=g).to(dev, torch.bfloat16)
    o.backward(d_o)
    ref = qkv.detach().float().requires_grad_(True)
    oref = torch.nn.functional.scaled_dot_product_attention(*(ref[:, :, i].transpose(1, 2) for i in range(3))).transpose(1, 2)
    oref.backward(d_o.float())
    assert rel(o, oref) <= 2.5e-3 and rel(qkv.grad, ref.grad) <= 2.5e-3


# ---- the model: forward and gradients against the goldens and the fp32 oracle ---------------------------------------------
@pytest.mark.parametrize("name", list(DIT_TYPE_CASES))
def test_forward_matches_oracle_and_golden(name, dev):
    cfg = DIT_TYPE_CASES[name]
    fx = json.load(open(os.path.join(GOLDEN, f"{name}.json")))
    gold = torch.load(os.path.join(GOLDEN, f"{name}.pt"))
    model, sd = build(cfg, dev)
    net = model.action_model.net
    assert (len(net.blocks), net.num_heads) == DIT_SIZES[cfg["dit_type"]]
    inp = synth.synth_inputs(cfg)
    dinp = {k: v.to(dev) for k, v in inp.items()}
    model.train()
    with torch.no_grad():
        out = model(dinp["image_primary"], dinp["image_wrist"], dinp["state"], dinp["text_token"],
                    action_label=dinp["action_label"], diffusion_noise=gold["diffusion_noise"].to(dev),
                    diffusion_timestep=gold["diffusion_timestep"].to(dev),
                    diffusion_drop_ids=gold["diffusion_drop_ids"].to(dev).long())
        ref = oracle_forward(sd, cfg, inp["image_primary"], inp["image_wrist"], inp["state"], inp["text_token"],
                                 action_label=inp["action_label"], diffusion_noise=gold["diffusion_noise"],
                                 diffusion_timestep=gold["diffusion_timestep"], diffusion_drop_ids=gold["diffusion_drop_ids"])
    assert abs(float(out[0]) - fx["loss_action"]) < 2e-2 * abs(fx["loss_action"])
    assert abs(float(out[0]) - float(ref["loss_action"])) < 2e-2 * abs(float(ref["loss_action"]))
    model.eval()
    with torch.no_grad():
        ot = model(dinp["image_primary"], dinp["image_wrist"], dinp["state"], dinp["text_token"], mode="test",
                   sample_noise=gold["sample_noise"].to(dev))
    assert rel(ot[0], gold["test_arm"]) < 5e-2
    assert rel(ot[1], gold["test_gripper"]) < 5e-2


@pytest.mark.parametrize("name", ["libero_dit_s", "libero_dit_l"])
def test_action_head_backward_matches_oracle(name, dev):
    """Gradients of the DiT action loss vs autograd through the fp32 oracle, same draws (the bar of
    test_model_gpu.py::test_flow_matching_head_backward)."""
    cfg = DIT_TYPE_CASES[name]
    gold = torch.load(os.path.join(GOLDEN, f"{name}.pt"))
    model, sd = build(cfg, dev)
    model.train()
    inp = synth.synth_inputs(cfg)
    dinp = {k: v.to(dev) for k, v in inp.items()}
    out = model(dinp["image_primary"], dinp["image_wrist"], dinp["state"], dinp["text_token"], action_label=dinp["action_label"],
                diffusion_noise=gold["diffusion_noise"].to(dev), diffusion_timestep=gold["diffusion_timestep"].to(dev),
                diffusion_drop_ids=gold["diffusion_drop_ids"].to(dev).long())
    out[0].float().backward()
    frozen = ("vision_encoder.", "clip_model.", "attention_mask", "position_embedding")
    osd = {k: v.clone() for k, v in sd.items()}
    for k, v in osd.items():
        if v.is_floating_point() and not any(f in k for f in frozen) or k == "transformer_backbone_position_embedding":
            v.requires_grad_(True)
    fwd = oracle_forward(osd, cfg, inp["image_primary"], inp["image_wrist"], inp["state"], inp["text_token"],
                             action_label=inp["action_label"], diffusion_noise=gold["diffusion_noise"],
                             diffusion_timestep=gold["diffusion_timestep"], diffusion_drop_ids=gold["diffusion_drop_ids"])
    fwd["loss_action"].backward()
    ref_loss = float(fwd["loss_action"].detach())
    assert abs(float(out[0]) - ref_loss) < 2e-2 * abs(ref_loss)
    last = DIT_SIZES[cfg["dit_type"]][0] - 1
    net = "action_model.net."
    probe = [net + f"blocks.{i}.{p}.weight" for i in (0, last) for p in ("attn.qkv", "mlp.fc2")] + \
            [net + p for p in ("x_embedder.linear.weight", "t_embedder.mlp.0.weight", "z_embedder.linear.weight",
                               "final_layer.linear.weight")] + ["action_pred_token", "transformer_backbone.h.1.mlp.c_proj.weight"]
    params = dict(model.named_parameters())
    worst = [(rel(params[k].grad, osd[k].grad), k) for k in probe]
    bad = [(e, k) for e, k in worst if not e < 6e-2]
    assert not bad, f"gradient mismatch: {bad}\nall: {sorted(worst, reverse=True)}"


# ---- rollouts ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["libero_dit_s", "libero_dit_l"])
def test_fused_sampler_matches_module_sampler_and_oracle(name, dev):
    """csrc/dit_sampler.cu at head_dim 96 (DiT-S) and at depth 24 / hidden 1024 (DiT-L) against the module path and the fp32
    oracle, with the criterion of test_rollout_gpu.py; the fused kernel is one launch."""
    from dreamvla_b200 import _lib as L
    from oracle import dreamvla_oracle as O
    cfg = DIT_TYPE_CASES[name]
    depth, heads = DIT_SIZES[cfg["dit_type"]]
    model = build(cfg, dev)[0].eval()
    sd = {k: v.detach().float().cpu() for k, v in model.state_dict().items() if k.startswith("action_model.")}
    g = torch.Generator().manual_seed(17)
    feat = (torch.randn(1, 3, 1024, generator=g) * 0.7).to(torch.bfloat16)
    noise = torch.randn(1, 3, 7, generator=g)
    with torch.no_grad():
        model.FUSED_SAMPLER = True
        model._ddim_actions(feat.to(dev), noise.to(dev), dev)          # first call: one-time set-up outside the count
        torch.cuda.synchronize()
        n0 = L.launch_count()
        a = model._ddim_actions(feat.to(dev), noise.to(dev), dev).float().cpu()
        assert L.launch_count() - n0 == 1, "the fused sampler did not run as one kernel"
        model.FUSED_SAMPLER = False
        b = model._ddim_actions(feat.to(dev), noise.to(dev), dev).float().cpu()
        unc = sd["action_model.net.z_embedder.uncondition"].unsqueeze(0).expand(1, 3, -1)
        z = torch.cat([feat.float(), unc], 0)
        x0 = torch.cat([noise.to(torch.bfloat16).float()] * 2, 0)

        def cfg_model(x, t):
            half = x[: len(x) // 2]
            out = O.dit_forward(sd, torch.cat([half, half], 0), t, z, depth=depth, heads=heads)
            cond, uncond = torch.split(out, len(out) // 2, dim=0)
            e = uncond + 1.5 * (cond - uncond)
            return torch.cat([e, e], 0)
        ref = O.Diffusion(100, use=set(range(0, 100, 10))).ddim_loop(cfg_model, x0)[:1]
    e_fused, e_mod = rel(a, ref), rel(b, ref)
    print(f"fused sampler {name}: vs oracle fused {e_fused:.3e} / module {e_mod:.3e}, fused vs module {rel(a, b):.3e}")
    assert torch.isfinite(a).all()
    assert e_fused <= e_mod + 5e-3, (e_fused, e_mod)


def test_incremental_rollout_dit_s_matches_full_window(dev):
    """DiT-S under the rollout engine: the incremental wrapper with prune=False gives the full window's actions bit for bit."""
    from dreamvla_b200.utils.eval_utils_calvin import ModelWrapper
    from tests.test_rollout_gpu import observations
    cfg = DIT_TYPE_CASES["libero_dit_s"]
    S = cfg["sequence_length"]
    model = build(cfg, dev)[0].eval()
    model.FUSED_SAMPLER = False          # the same sampler code on both sides (the fused kernel sums with fp32 atomics)
    text, obs = observations(S + 3, seed=11)
    full = ModelWrapper(model, history_len=S, device=dev, use_cuda_graph=True)
    inc = ModelWrapper(model, history_len=S, device=dev, use_cuda_graph=True, incremental=True, prune=False)
    g = torch.Generator().manual_seed(4)
    for i in range(len(obs)):
        noise = torch.randn(S, 3, 7, generator=g)
        a = full.step(*obs[i], text, sample_noise=noise)
        b = inc.step(*obs[i], text, sample_noise=noise)
        assert np.isfinite(b.astype(np.float32)).all()
        assert np.array_equal(a, b), (i, a, b)


# ---- train.py ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dit_type", ["DiT-S", "DiT-L"])
def test_train_py_dit_type(dev, tmp_path, dit_type):
    """train.main with --dit_type: the graphed step trains with finite losses, and the checkpoint holds the reference model's
    entries for that size (names and shapes recorded by tests/golden/make_golden_dit_types.py)."""
    from tests.test_train_entry_gpu import run
    ck = str(tmp_path)
    state, _ = run(["--dit_type", dit_type, "--cuda_graph", "--synthetic_steps", "3", "--num_epochs", "1", "--save_checkpoint",
                    "--save_checkpoint_path", ck, "--run_name", "t", "--start_save_checkpoint", "-1"])
    assert state.total_micro == 3
    assert getattr(state.model, "_dvla_graphed_step", None) is not None, "--cuda_graph did not capture"
    assert all(torch.isfinite(v).all() for v in state.last_terms.values())
    assert len(state.model.action_model.net.blocks) == {"DiT-S": 6, "DiT-L": 24}[dit_type]
    frozen = {n for n, p in state.model.named_parameters() if not p.requires_grad}
    del state
    # the checkpoint holds the trainable entries (train.py get_checkpoint, as the reference's train_utils.py:750-757)
    saved = torch.load(os.path.join(ck, "t", "0.pth"), map_location="cpu")["model_state_dict"]
    mine = {k[len("module."):]: list(v.shape) for k, v in saved.items()}
    ref = {k: v for k, v in json.load(open(os.path.join(GOLDEN, "dit_types_state.json")))[dit_type].items() if k not in frozen}
    assert any(k.startswith("action_model.net.blocks.") for k in mine)
    assert mine == ref, (sorted(set(mine) ^ set(ref)), [k for k in mine if k in ref and mine[k] != ref[k]])
