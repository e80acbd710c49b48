"""Pins the CPU oracle (oracle/dreamvla_oracle.py): (1) against the golden vectors generated from the unmodified
reference (tests/golden/*.pt), (2) against reference-side values recorded from the unmodified reference modules
(tests/golden/reference_checks.pt, written by tests/golden/make_golden_reference_checks.py)."""
import json
import os

import pytest
import torch

from oracle import dreamvla_oracle as O
from tests import synth

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
TOL = 2e-5   # fp32 vs fp32, different summation orders


def rel(a, b):
    return float((a.float() - b.float()).norm() / (b.float().norm() + 1e-12))


def template_state(cfg):
    """Shapes of every state_dict entry the oracle reads, derived from the fixture's config (no reference needed)."""
    from tests.state_template import build_template
    return build_template(cfg)


@pytest.mark.parametrize("name", list(synth.CASES) + list(synth.CPU_ONLY_CASES) + list(synth.FM_CASES))
def test_oracle_matches_reference_golden(name):
    cfg = {**synth.CASES, **synth.CPU_ONLY_CASES, **synth.FM_CASES}[name]
    fx = json.load(open(os.path.join(GOLDEN, f"{name}.json")))
    gold = torch.load(os.path.join(GOLDEN, f"{name}.pt"))
    torch.set_num_threads(min(8, os.cpu_count() or 1))
    sd = synth.synth_state_dict(template_state(cfg), cfg["weight_seed"])
    inp = synth.synth_inputs(cfg)
    with torch.no_grad():
        out = O.dreamvla_forward(sd, cfg, inp["image_primary"], inp["image_wrist"], inp["state"], inp["text_token"],
                                 action_label=inp["action_label"], mode="train",
                                 diffusion_noise=gold.get("diffusion_noise"),
                                 diffusion_timestep=gold.get("diffusion_timestep"),
                                 diffusion_drop_ids=gold.get("diffusion_drop_ids"))
    for k in ("image_pred", "depth_pred", "traj_pred", "dino_pred", "sam_pred"):
        if k + "_sub" in gold:
            assert list(out[k].shape) == fx[k + "_shape"]
            assert rel(synth.subsample(out[k]), gold[k + "_sub"]) < TOL, k
    assert rel(synth.subsample(out["vit_primary"]), gold["vit_primary_sub"]) < TOL
    assert rel(synth.subsample(out["resampler_primary"]), gold["resampler_primary_sub"]) < TOL
    if cfg["use_dit_head"]:
        assert abs(float(out["loss_action"]) - fx["loss_action"]) < 1e-4 * abs(fx["loss_action"])
        with torch.no_grad():
            o2 = O.dreamvla_forward(sd, cfg, inp["image_primary"], inp["image_wrist"], inp["state"], inp["text_token"],
                                    mode="test", sample_noise=gold["sample_noise"])
        assert rel(o2["arm_pred_action"], gold["test_arm"]) < TOL
        assert rel(o2["gripper_pred_action"], gold["test_gripper"]) < TOL
    else:
        assert rel(synth.subsample(out["arm_pred_action"]), gold["arm_sub"]) < TOL
        assert rel(synth.subsample(out["gripper_pred_action"]), gold["gripper_sub"]) < TOL
    # the ViT token permutation of the reference (vit_mae.py:157-182) is output-invariant at fp32 noise level
    assert fx["perm_invariance_rel"] < 5e-6 and fx["perm_cls_rel"] < 5e-6


def test_state_template_matches_reference_keys():
    """The shape template has exactly the reference's state_dict entries (minus the dead MAE decoder), as recorded from the
    reference model by tests/golden/make_golden_reference_checks.py."""
    ref = torch.load(os.path.join(GOLDEN, "reference_checks.pt"))["state_keys"]
    tmpl = {k: tuple(v.shape) for k, v in template_state(synth.CASES["calvin_allheads"]).items()}
    assert ref == tmpl


# ----------------------------------------------------------------------------------------------------------------------
# train step: the oracle's loss half + the reference's accumulate / clip / step rules, pinned to the golden that
# tests/golden/make_golden_step.py recorded from the reference's OWN step loop (utils/train_utils.py:59-726)
# ----------------------------------------------------------------------------------------------------------------------
def step_fixture(name="step_calvin_accum2"):
    fx = json.load(open(os.path.join(GOLDEN, f"{name}.json")))
    gold = torch.load(os.path.join(GOLDEN, f"{name}.pt"))
    return fx, gold


def step_batches(fx, cfg):
    from dreamvla_b200.utils.train_utils import StepConfig, synthetic_batch
    scfg = StepConfig(sequence_length=cfg["sequence_length"], future_steps=3)
    heads = dict(depth=True, dino=True, sam=True, traj=True, flow_mask=True)
    return [synthetic_batch(scfg, fx["case"]["batch"], "cpu", seed=fx["case"]["data_seed"] + i, heads=heads,
                            dtype=torch.float32) for i in range(fx["case"]["num_batches"])]


def oracle_micro_step(sd, cfg, b, gold, i, flow_as_mask=True):
    """Forward + total loss of one micro-batch, as train_utils.py:124-170,585 prepares the inputs (CALVIN gripper remap,
    sliding-window action labels)."""
    S, aps = cfg["sequence_length"], cfg["action_pred_steps"]
    states = torch.cat([b["states"][..., :6], b["states"][..., -1:]], dim=-1)
    states[..., 6:] = (states[..., 6:] + 1) // 2
    actions = b["actions"].clone()
    actions[..., 6:] = (actions[..., 6:] + 1) // 2
    labels = torch.cat([actions[:, j:S + j].unsqueeze(-2) for j in range(aps)], dim=-2)
    text = b["text"].unsqueeze(1).repeat(1, S, 1)
    fwd = O.dreamvla_forward(sd, cfg, b["images_primary"][:, :S], b["images_wrist"][:, :S], states[:, :S], text,
                             action_label=labels[:, :S], diffusion_noise=gold[f"noise_{i}"],
                             diffusion_timestep=gold[f"timestep_{i}"], diffusion_drop_ids=gold[f"drop_{i}"])
    return O.train_losses(dict(cfg, future_steps=3, flow_as_mask=flow_as_mask), fwd, b)


def test_oracle_train_step_matches_reference_loop():
    """Loss half of the oracle (patchify / normalise / flow masks / SiLog / cosine / pixel-unshuffle, weights of :585) and
    the reference's accumulation rules -- all-micro-step clip of the ACCUMULATED gradient (:599-600), optimiser step on
    the boundary and on the last batch (:602-604) -- against numbers recorded from the reference's own loop."""
    fx, gold = step_fixture()
    cfg = dict(synth.CASES[fx["case"]["model"]])
    accum = fx["case"]["accum"]
    torch.set_num_threads(min(8, os.cpu_count() or 1))
    sd = synth.synth_state_dict(template_state(cfg), cfg["weight_seed"])
    sd["depth_decoder_pred.bias"] = sd["depth_decoder_pred.bias"] + fx["depth_bias_shift"]
    frozen = ("vision_encoder.", "clip_model.", "attention_mask", "position_embedding")
    train = [k for k, v in sd.items() if v.is_floating_point() and (not any(f in k for f in frozen)
                                                                     or k == "transformer_backbone_position_embedding")]
    for k in train:
        sd[k].requires_grad_(True)
    batches = step_batches(fx, cfg)
    acc = {k: torch.zeros_like(sd[k]) for k in train}
    step_no = 0
    for i in range(2):                      # micro-steps 1 and 2 run on the initial weights (first optimiser step after 2)
        ol = oracle_micro_step(sd, cfg, batches[i], gold, i)
        loss = ol["loss"] / accum
        assert abs(float(loss) - fx["micro_losses"][i]) < 2e-5 * abs(fx["micro_losses"][i]), (i, float(loss))
        grads = torch.autograd.grad(loss, [sd[k] for k in train], allow_unused=True)
        for k, g in zip(train, grads):
            if g is not None:
                acc[k] += g
        norm = torch.sqrt(sum((g.double() ** 2).sum() for g in acc.values())).float()
        assert abs(float(norm) - fx["accumulated_grad_norms"][i]) < 1e-4 * fx["accumulated_grad_norms"][i], (i, float(norm))
        coef = min(1.0, 0.1 / (float(norm) + 1e-6))                     # clip_grad_norm_ semantics
        for g in acc.values():
            g.mul_(coef)
        if i + 1 in fx["optimizer_steps_after_micro"]:
            for k in fx["probe"]:
                assert rel(synth.subsample(acc[k], 2048), gold[f"grad{step_no}:{k}"]) < 2e-4, (k, step_no)
            step_no += 1
    # the individual terms the loop logs on the boundary (wandb dict, already multiplied back by accum)
    log = fx["wandb_loss_logs"][0]
    for mine, theirs in (("loss_action", "loss_arm_action"), ("loss_image", "loss_image"), ("loss_depth", "loss_depth"),
                         ("loss_dino", "loss_dino_feat"), ("loss_sam", "loss_sam_feat"), ("loss_traj", "loss_pred_trajectory")):
        # logging quirk of the reference: `loss_pred_depth` is logged times accum without having been divided by it
        # (train_utils.py:592 assigns the divided value to `loss_depth`, :716 logs `loss_pred_depth`)
        want = log[theirs] / accum if mine == "loss_depth" else log[theirs]
        assert abs(float(ol[mine]) - want) < 2e-5 * abs(want) + 1e-7, (mine, float(ol[mine]), want)
    assert abs(float(ol["loss"]) - log["loss_calvin"]) < 2e-5 * abs(log["loss_calvin"])
    assert fx["optimizer_steps_after_micro"] == [2, 3] and len(fx["micro_losses"]) == 3    # last-batch rule fired


def test_oracle_loss_helpers_match_reference_functions():
    """patchify / normalize_patchfied_image / unpatchify (utils/train_utils.py:37-57,783-799) and SiLogLoss
    (utils/sigloss.py:11-15) of the UNMODIFIED reference vs the oracle's restatements and the product's.  The reference's
    outputs on these seeded inputs are stored (sampled elements + float64 sums) by tests/golden/make_golden_reference_checks.py."""
    from dreamvla_b200.utils import train_utils as P
    ref = torch.load(os.path.join(GOLDEN, "reference_checks.pt"))["loss_helpers"]

    def same(t, r):
        flat = t.reshape(-1)
        return (list(t.shape) == r["shape"] and torch.equal(flat[r["idx"]], r["val"])
                and float(flat.double().sum()) == r["sum"])

    g = torch.Generator().manual_seed(3)
    imgs = torch.randn(3, 3, 224, 224, generator=g)
    x = O.patchify(imgs, 16)
    assert same(x, ref["patchify"]) and torch.equal(P.patchify(imgs, 16), x)
    assert same(O.normalize_patchfied_image(x), ref["normalize"]) and same(P.normalize_patchfied_image(x), ref["normalize"])
    pt = torch.rand(2, 1, 196, 256, generator=g) + 0.1
    assert same(O.unpatchify(pt), ref["unpatchify"]) and same(P.unpatchify(pt), ref["unpatchify"])
    tgt = torch.rand(2, 1, 1, 224, 224, generator=g) * 4 + 0.1
    assert abs(float(O.silog(O.unpatchify(pt), tgt)) - ref["silog"]) < 1e-7
    # the product permutes the LABEL instead of un-permuting the prediction (patchify_map): same SiLog value
    lab = P.patchify_map(tgt.flatten(0, 1), 16)
    assert abs(float(O.silog(pt[:, 0], lab)) - ref["silog"]) < 1e-6
