"""Flow-matching (`--use_fm`) rollouts on the fused sampler (csrc/dit_sampler.cu, Euler integrator) on the GPU: the kernel
against the module path (FMDiffusion.ddim_sample_loop over the DiT modules) and an fp32 oracle Euler loop for DiT-S, DiT-B and
DiT-L; the start-state draw; and both rollout wrappers, incremental under CUDA graphs, on the fused path."""
import numpy as np
import pytest
import torch

from tests import synth
from tests.dit_types import DIT_SIZES, DIT_TYPE_CASES

pytestmark = pytest.mark.gpu

# one flow-matching model per action-head size; DiT-L has no golden and needs none (the oracle runs here)
FM_SIZES = {
    "DiT-S": DIT_TYPE_CASES["libero_fm_dit_s"],
    "DiT-B": synth.FM_CASES["libero_fm"],
    "DiT-L": dict(synth.FM_CASES["libero_fm"], dit_type="DiT-L", weight_seed=81, input_seed=82, draw_seed=83),
}


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return float((a - b).norm() / (b.norm() + 1e-12))


def build(cfg, dev):
    from tests.test_dit_type_gpu import build as build_dit
    return build_dit(cfg, dev)[0].eval()


def oracle_fm_loop(sd, feat, start, depth, heads, n_steps=10):
    """FMDiffusion.ddim_sample_loop (respace.py:122-156) in fp32 over oracle.dit_forward: guidance scale 1.0 over both branches,
    t = i / n_steps, final += (1 / n_steps) u.  feat [bs, 3, token], start [bs, 3, 7] -> [bs, 3, 7]."""
    from oracle import dreamvla_oracle as O
    bs = feat.shape[0]
    unc = sd["action_model.net.z_embedder.uncondition"].unsqueeze(0).expand(bs, 3, -1)
    z = torch.cat([feat.float(), unc], 0)
    final = torch.cat([start.float()] * 2, 0)
    for i in range(n_steps):
        t = torch.full((final.shape[0],), float(i)) / n_steps
        half = final[: len(final) // 2]
        out = O.dit_forward(sd, torch.cat([half, half], 0), t, z, depth=depth, heads=heads)
        cond, uncond = torch.split(out, len(out) // 2, dim=0)
        u = uncond + 1.0 * (cond - uncond)
        final = final + (1 / n_steps) * torch.cat([u, u], 0)
    return final[:bs]


@pytest.mark.parametrize("dit_type", list(FM_SIZES))
def test_fused_fm_sampler_matches_module_sampler_and_oracle(dit_type, dev):
    """The criterion of test_rollout_gpu.py: the fused kernel is no further from the fp32 oracle than the module path, + 5e-3."""
    from dreamvla_b200 import _lib as L
    cfg = FM_SIZES[dit_type]
    depth, heads = DIT_SIZES[dit_type]
    model = build(cfg, dev)
    net = model.action_model.net
    assert model.use_fm and (len(net.blocks), net.num_heads) == (depth, heads)
    sd = {k: v.detach().float().cpu() for k, v in model.state_dict().items() if k.startswith("action_model.")}
    g = torch.Generator().manual_seed(23)
    feat = (torch.randn(1, 3, 1024, generator=g) * 0.7).to(torch.bfloat16)
    start = torch.randn(1, 3, 7, generator=g)
    with torch.no_grad():
        model.FUSED_SAMPLER = True
        model._ddim_actions(feat.to(dev), start.to(dev), dev)          # first call: one-time set-up outside the count
        torch.cuda.synchronize()
        n0 = L.launch_count()
        a = model._ddim_actions(feat.to(dev), start.to(dev), dev).float().cpu()
        assert L.launch_count() - n0 == 1, "the fused FM sampler did not run as one kernel"
        model.FUSED_SAMPLER = False
        b = model._ddim_actions(feat.to(dev), start.to(dev), dev).float().cpu()
        ref = oracle_fm_loop(sd, feat, start, depth, heads)
    e_fused, e_mod = rel(a, ref), rel(b, ref)
    print(f"fused FM sampler {dit_type}: vs oracle fused {e_fused:.3e} / module {e_mod:.3e}, fused vs module {rel(a, b):.3e}")
    assert torch.isfinite(a).all()
    assert e_fused <= e_mod + 5e-3, (e_fused, e_mod)


def test_fused_fm_sampler_draws_the_start_state_as_the_module_path(dev):
    """With no injected start state both paths draw torch.randn(2 bs, steps, 7) on the device: switching FUSED_SAMPLER does not
    shift the CUDA generator."""
    model = build(FM_SIZES["DiT-B"], dev)
    feat = (torch.randn(1, 3, 1024, generator=torch.Generator().manual_seed(29)) * 0.7).to(dev, torch.bfloat16)
    torch.cuda.manual_seed(1234)
    s0 = torch.cuda.get_rng_state()
    states, outs = [], []
    with torch.no_grad():
        for fused in (True, False):
            torch.cuda.set_rng_state(s0)
            model.FUSED_SAMPLER = fused
            outs.append(model._ddim_actions(feat, None, dev).float().cpu())
            states.append(torch.cuda.get_rng_state())
    assert not torch.equal(states[0], s0)
    assert torch.equal(states[0], states[1])
    assert torch.isfinite(outs[0]).all()
    print(f"fused vs module FM sampler from the same draw: rel {rel(outs[0], outs[1]):.3e}")


@pytest.mark.parametrize("suite", ["calvin", "libero"])
def test_fm_rollout_wrappers_take_the_fused_sampler(suite, dev, monkeypatch):
    """An FM model through the rollout wrapper, incremental under CUDA graphs, S + 2 steps with fixed start states: the graphs
    are captured on the fused path (one sampler launch inside each capture) and the arm actions agree with a FUSED_SAMPLER =
    False run to the bar of the pruned incremental test (1e-2 rel-L2)."""
    from dreamvla_b200 import _lib as L
    from tests.test_rollout_gpu import observations
    cfg = FM_SIZES["DiT-B"]
    S = cfg["sequence_length"]
    model = build(cfg, dev)
    calls = []
    orig = L.dit_fm_sample

    def spy(*args, **kwargs):
        n0 = L.launch_count()
        out = orig(*args, **kwargs)
        calls.append((model.FUSED_SAMPLER, torch.cuda.is_current_stream_capturing(), L.launch_count() - n0))
        return out
    monkeypatch.setattr(L, "dit_fm_sample", spy)

    if suite == "calvin":
        from dreamvla_b200.utils.eval_utils_calvin import ModelWrapper
        make = lambda: ModelWrapper(model, history_len=S, device=dev, use_cuda_graph=True, incremental=True)   # noqa: E731
    else:
        from dreamvla_b200.utils.eval_utils_libero import ModelWrapper
        make = lambda: ModelWrapper(model, history_len=S, device=dev, use_cuda_graph=True, incremental=True)   # noqa: E731
    wrappers = {True: make(), False: make()}
    text, obs = observations(S + 2, seed=31)
    g = torch.Generator().manual_seed(37)
    arms = {True: [], False: []}
    for i in range(S + 2):
        noise = torch.randn(S, 3, 7, generator=g)
        pose = (torch.randn(3, generator=g).numpy() * 0.3, torch.randn(4, generator=g).numpy(), torch.rand(2, generator=g).numpy() * 0.04)
        for fused in (True, False):
            model.FUSED_SAMPLER = fused
            w = wrappers[fused]
            if suite == "calvin":
                a = w.step(*obs[i], text, sample_noise=noise)
            else:
                a = w.step(obs[i][0], obs[i][1], *pose, text, i, sample_noise=noise)
            a = a.astype(np.float32)
            assert np.isfinite(a).all(), (fused, i, a)
            arms[fused].append(a[:6])
    captured = [c for c in calls if c[1]]
    assert captured, "no sampler call was captured into a graph"
    assert all(fused and n == 1 for fused, _, n in captured), calls        # one launch, on the fused model only
    assert not any(not fused for fused, _, _ in calls), calls
    assert len(captured) == len(wrappers[True]._act_graphs) == S             # one graph per selected timestep 0 .. S-1
    a, b = np.stack(arms[True]), np.stack(arms[False])
    err = float(np.linalg.norm(a - b) / (np.linalg.norm(b) + 1e-12))
    print(f"FM rollout [{suite}] fused vs module arm actions rel-L2 {err:.3e}")
    assert err <= 1e-2, err
