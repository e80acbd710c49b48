"""The fused sampler's multi-sequence bucket (csrc/dit_sampler.cu, 2 .. 8 sequences on tensor-core GEMMs) on the GPU, for
DiT-S, DiT-B and DiT-L under DDIM and flow matching: against the module sampler at the same batch and the fp32 oracle loop,
with the criterion of the batch-1 tests (test_rollout_gpu.py): the fused kernel is no further from the oracle than the module
path, + 5e-3."""
import pytest
import torch

from tests import synth
from tests.dit_types import DIT_SIZES, DIT_TYPE_CASES
from tests.test_fm_sampler_gpu import FM_SIZES, oracle_fm_loop

pytestmark = pytest.mark.gpu

DDIM_SIZES = {"DiT-S": DIT_TYPE_CASES["libero_dit_s"], "DiT-B": synth.CASES["libero_dit"], "DiT-L": DIT_TYPE_CASES["libero_dit_l"]}


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return float((a - b).norm() / (b.norm() + 1e-12))


def oracle_ddim_loop(sd, feat, noise, depth, heads):
    from oracle import dreamvla_oracle as O
    bs = feat.shape[0]
    unc = sd["action_model.net.z_embedder.uncondition"].unsqueeze(0).expand(bs, 3, -1)
    z = torch.cat([feat.float(), unc], 0)
    x0 = torch.cat([noise.to(torch.bfloat16).float()] * 2, 0)

    def cfg_model(x, t):
        half = x[: len(x) // 2]
        out = O.dit_forward(sd, torch.cat([half, half], 0), t, z, depth=depth, heads=heads)
        cond, uncond = torch.split(out, len(out) // 2, dim=0)
        e = uncond + 1.5 * (cond - uncond)
        return torch.cat([e, e], 0)
    return O.Diffusion(100, use=set(range(0, 100, 10))).ddim_loop(cfg_model, x0)[:bs]


@pytest.mark.parametrize("integrator", ["ddim", "fm"])
@pytest.mark.parametrize("dit_type", list(DIT_SIZES))
def test_multi_sequence_fused_sampler_matches_module_sampler_and_oracle(dit_type, integrator, dev):
    from dreamvla_b200 import _lib as L
    from tests.test_dit_type_gpu import build
    cfg = (DDIM_SIZES if integrator == "ddim" else FM_SIZES)[dit_type]
    depth, heads = DIT_SIZES[dit_type]
    model = build(cfg, dev)[0].eval()
    model.FUSED_SAMPLER_MAX_BATCH = 8                  # the kernel's whole range, above the crossover rollouts use
    assert model.use_fm == (integrator == "fm")
    sd = {k: v.detach().float().cpu() for k, v in model.state_dict().items() if k.startswith("action_model.")}
    g = torch.Generator().manual_seed(29)
    worst = []
    for n in (2, 4, 8):
        feat = (torch.randn(n, 3, 1024, generator=g) * 0.7).to(torch.bfloat16)
        noise = torch.randn(n, 3, 7, generator=g)
        with torch.no_grad():
            model.FUSED_SAMPLER = True
            model._ddim_actions(feat.to(dev), noise.to(dev), dev, multi=True)     # one-time set-up outside the count
            torch.cuda.synchronize()
            n0 = L.launch_count()
            a = model._ddim_actions(feat.to(dev), noise.to(dev), dev, multi=True).float().cpu()
            assert L.launch_count() - n0 == 1, "the fused sampler did not run as one kernel"
            model.FUSED_SAMPLER = False
            b = model._ddim_actions(feat.to(dev), noise.to(dev), dev, multi=True).float().cpu()
            ref = (oracle_ddim_loop(sd, feat, noise, depth, heads) if integrator == "ddim"
                   else oracle_fm_loop(sd, feat, noise, depth, heads))
        e_fused, e_mod = rel(a, ref), rel(b, ref)
        worst.append((n, e_fused, e_mod, rel(a, b)))
        assert torch.isfinite(a).all()
        assert e_fused <= e_mod + 5e-3, worst
    print(f"{dit_type} {integrator}: " + "; ".join(f"N={n}: vs oracle fused {ef:.3e} / module {em:.3e}, fused vs module {d:.3e}"
                                                   for n, ef, em, d in worst))
