"""`--precision fp32`: fp32 master weights updated by dvla_adamw_master, with the bf16 working copy the kernels read rounded
from them once per optimiser step.  Checked against torch.optim.AdamW on fp32 parameters, against the update the reference's
own fp32 loop made (tests/golden/step_calvin_accum2), and through train.py's checkpoint writer and resume."""
import copy
import json
import os

import pytest
import torch

from tests import synth
from tests.test_train_entry_gpu import FLAGS

pytestmark = pytest.mark.gpu

FP32 = ["--precision", "fp32", "--bf16_module", "vision_encoder"]


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def build(cfg_name, dev, lr, wd, sd_edit=None):
    """The synth model of `cfg_name` in bf16 on `dev` (dropout off) and the fp32 state dict it was loaded from."""
    from dreamvla_b200.models import DreamVLA
    cfg = synth.CASES[cfg_name]
    torch.manual_seed(0)
    m = DreamVLA(finetune_type="calvin", clip_device="cpu", vit_checkpoint_path=None, **synth.ctor_kwargs(cfg))
    sd = synth.synth_state_dict(m.state_dict(), cfg["weight_seed"])
    if sd_edit:
        sd_edit(sd)
    m.load_state_dict(sd)
    m = m.bfloat16().to(dev)
    m._init_model_type()
    m.train()
    gp = m.transformer_backbone
    gp.embd_pdrop = 0.0
    for blk in gp.h:
        blk.attn.attn_pdrop = blk.attn.resid_pdrop = blk.mlp.resid_pdrop = 0.0
    return m, cfg, sd


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def test_master_adamw_matches_torch_over_100_steps(dev):
    """100 clipped AdamW steps (lr 1e-5, wd 1e-2) on seeded bf16 gradients: the fp32 masters follow torch.optim.AdamW on
    fp32 parameters; the bf16 working copy is exactly the rounded master; a bf16-only run loses most of the update."""
    from dreamvla_b200.utils.train_utils import StepConfig, TrainStep
    lr, wd = 1e-5, 1e-2
    m, cfg, sd = build("pretrain_mlp", dev, lr, wd)
    scfg = StepConfig(sequence_length=cfg["sequence_length"], use_dit_head=cfg["use_dit_head"], loss_action=True,
                      loss_image=cfg["obs_pred"], learning_rate=lr, weight_decay=wd)
    m_bf = copy.deepcopy(m)
    fp = TrainStep(m, scfg, master=sd).flat
    bf = TrainStep(m_bf, scfg).flat
    assert fp.P32 is not None and bf.P32 is None
    P0 = fp.P32.clone()
    assert torch.equal(fp.P, P0.to(torch.bfloat16)) and torch.equal(bf.P, fp.P)
    ref = P0.clone().requires_grad_(True)
    opt = torch.optim.AdamW([ref], lr=lr, weight_decay=wd, betas=(0.9, 0.999), eps=1e-8)
    gen = torch.Generator(device=dev).manual_seed(2024)
    clipped = 0
    for it in range(100):
        g = (torch.randn(fp.n, device=dev, generator=gen) * (1e-3 if it % 2 else 1e-5)).to(torch.bfloat16)
        ref.grad = g.float()
        clipped += float(torch.nn.utils.clip_grad_norm_([ref], scfg.max_grad_norm)) > scfg.max_grad_norm
        opt.step()
        for f in (fp, bf):
            f.G.copy_(g)
            f.optimizer_step(scfg, lr, 1)
        assert torch.equal(fp.P, fp.P32.to(torch.bfloat16)), it
        assert fp.G.abs().max().item() == 0 and bf.G.abs().max().item() == 0, it
    assert 0 < clipped < 100                      # both sides of the clip are exercised
    want = ref.detach() - P0
    e32 = rel(fp.P32 - P0, want)
    e16 = rel(bf.P.float() - P0, want)
    st = opt.state[ref]
    e_m, e_v = rel(fp.m, st["exp_avg"]), rel(fp.v, st["exp_avg_sq"])
    # torch scales g^2 by 1 - beta2 computed in double (0.001) but decays by float(0.999); the kernel uses 1 - float(0.999),
    # 1.29e-5 smaller.  The bias-corrected second moment -- what the update divides by -- carries the same factor in the
    # correction and agrees far closer; the raw moment is held to that constant factor.
    b2 = torch.tensor(0.999, dtype=torch.float32).double()
    bc2_kernel, bc2_torch = 1.0 - b2 ** 100, 1.0 - 0.999 ** 100
    e_vhat = rel(fp.v.double() / bc2_kernel, st["exp_avg_sq"].double() / bc2_torch)
    print(f"100 steps: update rel-L2 vs torch fp32 AdamW: fp32 masters {e32:.3e}, bf16 parameters {e16:.3e}; "
          f"moments m {e_m:.2e}, v {e_v:.2e}, bias-corrected v {e_vhat:.2e}")
    assert e32 <= 1e-5
    assert e_m <= 1e-5 and e_vhat <= 1e-5 and e_v <= 1.29e-5 + 1e-6
    assert e16 >= 10 * e32


def test_accumulation_follows_the_reference_loop_fp32(dev):
    """test_train_step_gpu.test_accumulation_follows_the_reference_loop with fp32 master weights, plus the parameter update
    itself: AdamW is elementwise, so the reference's update of the probe elements follows from the golden's recorded
    accumulated gradients and the synth initial weights; the P32 delta is compared with it at both optimiser steps (a bf16
    parameter buffer rounds this lr-1e-7 update away entirely: its error is 1.0).  Measured on an H100 80GB HBM3 (700 W):
    rel-L2 8.7e-2 after the first optimiser step, 5.4e-2 after the second; the bound is 1.5x the larger."""
    from dreamvla_b200.utils.train_utils import StepConfig, TrainStep, synthetic_batch
    gdir = os.path.join(os.path.dirname(__file__), "golden")
    fx = json.load(open(os.path.join(gdir, "step_calvin_accum2.json")))
    gold = torch.load(os.path.join(gdir, "step_calvin_accum2.pt"))
    case = fx["case"]

    def shift(sd):
        sd["depth_decoder_pred.bias"] = sd["depth_decoder_pred.bias"] + fx["depth_bias_shift"]
    m, cfg, sd = build(case["model"], dev, case["lr"], case["weight_decay"], shift)
    scfg = StepConfig(sequence_length=cfg["sequence_length"], future_steps=3, use_dit_head=True, loss_image=True, loss_depth=True,
                      loss_dino_feat=True, loss_sam_feat=True, loss_trajectory=True, flow_as_mask=True,
                      gradient_accumulation_steps=case["accum"], learning_rate=case["lr"], weight_decay=case["weight_decay"])
    step = TrainStep(m, scfg, master=sd)
    masters = step.flat.master_state_dict()
    probe = fx["probe"]
    assert all(k in step.flat.names for k in probe)
    # the reference's AdamW on the probe elements (torch.optim.AdamW, fp32, no clip: the recorded gradients are clipped)
    w0 = torch.cat([synth.subsample(sd[k], 2048) for k in probe])
    ref = w0.clone().requires_grad_(True)
    opt = torch.optim.AdamW([ref], lr=case["lr"], weight_decay=case["weight_decay"])
    heads = dict(depth=True, dino=True, sam=True, traj=True, flow_mask=True)
    params = dict(m.named_parameters())
    report, step_no, update_err = [], 0, []
    for i in range(case["num_batches"]):
        batch = synthetic_batch(scfg, case["batch"], dev, seed=case["data_seed"] + i, heads=heads, dtype=torch.float32)
        batch = {k: (v.to(torch.bfloat16) if v.is_floating_point() else v) for k, v in batch.items()}
        draws = dict(diffusion_noise=gold[f"noise_{i}"].to(dev), diffusion_timestep=gold[f"timestep_{i}"].to(dev),
                     diffusion_drop_ids=gold[f"drop_{i}"].to(dev).long())
        boundary = (i + 1) in fx["optimizer_steps_after_micro"]
        step.flat.lr.fill_(case["lr"])
        loss = float(step.micro_step(batch, boundary=boundary, draws=draws))
        norm = float(step.flat.sumsq.sqrt())
        e_loss = abs(loss - fx["micro_losses"][i]) / abs(fx["micro_losses"][i])
        e_norm = abs(norm - fx["accumulated_grad_norms"][i]) / fx["accumulated_grad_norms"][i]
        report.append(f"micro {i}: loss {loss:.5f} vs {fx['micro_losses'][i]:.5f} (rel {e_loss:.2e}); "
                      f"|G| {norm:.3f} vs {fx['accumulated_grad_norms'][i]:.3f} (rel {e_norm:.2e})")
        assert e_loss < (2e-2 if i < 2 else 6e-2) and e_norm < (3e-2 if i < 2 else 8e-2), report
        if boundary:
            worst = max((float((synth.subsample(params[k].grad, 2048).cpu() - gold[f"grad{step_no}:{k}"]).norm()
                               / gold[f"grad{step_no}:{k}"].norm()), k) for k in probe)
            report.append(f"optimizer step {step_no}: worst accumulated-clipped-gradient rel-L2 {worst[0]:.3e} ({worst[1]})")
            assert worst[0] < (6e-2 if step_no == 0 else 1.5e-1), report
            total = float(torch.sqrt(step.flat.G.float().pow(2).sum()))
            assert abs(total - 0.1) < 2e-3, total
            step.flat.optimizer_step(scfg, None, 1, preclipped=step.per_micro_clip)
            assert step.flat.G.abs().max().item() == 0
            assert torch.equal(step.flat.P, step.flat.P32.to(torch.bfloat16))
            ref.grad = torch.cat([gold[f"grad{step_no}:{k}"] for k in probe]).float()
            opt.step()
            got = torch.cat([synth.subsample(masters[k], 2048).cpu() for k in probe]) - w0
            e = rel(got, ref.detach() - w0)
            update_err.append(e)
            report.append(f"optimizer step {step_no}: P32 update rel-L2 vs the reference's update {e:.3e} (bf16 parameters: 1.0)")
            step_no += 1
    print("\n".join(report))
    assert step_no == 2
    assert max(update_err) <= 0.13, report


def run(extra):
    import train
    from dreamvla_b200.utils.arguments_utils import get_parser
    args = get_parser().parse_args(FLAGS + FP32 + extra)
    return train.main(args), args


def test_fp32_checkpoint_keeps_the_loaded_values(dev, tmp_path):
    """A model_state_dict whose fp32 values bf16 cannot represent, resumed with nothing left to train, is written back by
    get_checkpoint in fp32 and bit-equal, for the parameters the step trains and for those it does not."""
    import train
    from dreamvla_b200.models import DreamVLA
    from dreamvla_b200.utils.arguments_utils import get_parser, model_kwargs
    a = get_parser().parse_args(FLAGS + FP32)
    cpu_model = DreamVLA(finetune_type=a.finetune_type, clip_device="cpu", vit_checkpoint_path=None, **model_kwargs(a))
    cpu_model.clip_model.requires_grad_(False)
    cpu_model.vision_encoder.requires_grad_(False)
    g = torch.Generator().manual_seed(11)
    loaded = {"module." + n: p.detach().float() + torch.randn(p.shape, generator=g) * 1e-3
              for n, p in cpu_model.named_parameters() if p.requires_grad}
    del cpu_model
    exact = sum(int((v == v.to(torch.bfloat16).float()).sum()) for v in loaded.values())
    assert exact < 1e-3 * sum(v.numel() for v in loaded.values())
    path = str(tmp_path / "in.pth")
    torch.save({"epoch": 0, "model_state_dict": loaded, "lr_scheduler_state_dict": {"step_idx": 0}}, path)
    state, _ = run(["--synthetic_steps", "1", "--num_epochs", "1", "--resume_from_checkpoint", path])
    assert state.total_micro == 0 and state.flat.P32 is not None
    assert torch.equal(state.flat.P, state.flat.P32.to(torch.bfloat16))
    assert len(state.flat.master_rest) > 0            # parameters the step does not train are part of the round trip
    wrapped = train._ModuleWrapper(state.model)
    sd = train.get_checkpoint(wrapped, state)
    assert set(sd) == set(train.get_checkpoint(wrapped))                    # same keys as the bf16 writer
    trainable = {"module." + n for n, p in state.model.named_parameters() if p.requires_grad}
    assert trainable == set(loaded)
    for k, v in loaded.items():
        assert sd[k].dtype == torch.float32 and torch.equal(sd[k].cpu(), v), k


def test_fp32_resume_restores_masters_and_moments(dev, tmp_path):
    ck = str(tmp_path)
    s1, _ = run(["--synthetic_steps", "2", "--num_epochs", "1", "--save_checkpoint", "--save_checkpoint_path", ck,
                 "--run_name", "t", "--start_save_checkpoint", "-1"])
    path = os.path.join(ck, "t", "0.pth")
    saved = torch.load(path, map_location="cpu")
    trainable = {"module." + n for n, p in s1.model.named_parameters() if p.requires_grad}
    assert all(saved["model_state_dict"][k].dtype == torch.float32 for k in trainable)
    assert saved["optimizer_state_dict"]["format"] == "dvla_flat_adamw_v1"
    P32, m1, v1, n1 = s1.flat.P32.clone(), s1.flat.m.clone(), s1.flat.v.clone(), s1.flat.step_count.clone()
    assert float(n1) == 2.0 and not torch.equal(P32.to(torch.bfloat16).float(), P32)
    del s1
    s2, _ = run(["--synthetic_steps", "1", "--num_epochs", "1", "--resume_from_checkpoint", path])
    assert s2.total_micro == 0
    assert torch.equal(s2.flat.P32, P32) and torch.equal(s2.flat.m, m1) and torch.equal(s2.flat.v, v1)
    assert torch.equal(s2.flat.step_count, n1)


def test_fp32_graph_with_accumulation(dev):
    state, _ = run(["--synthetic_steps", "5", "--gradient_accumulation_steps", "2", "--cuda_graph"])
    assert state.total_micro == 5 and float(state.flat.step_count) == 3.0
    assert getattr(state.model, "_dvla_graphed_step", None) is not None, "--cuda_graph did not capture"
    assert all(torch.isfinite(v).all() for v in state.last_terms.values())
    assert float(state.flat.G.abs().max()) == 0.0
    assert torch.equal(state.flat.P, state.flat.P32.to(torch.bfloat16))
