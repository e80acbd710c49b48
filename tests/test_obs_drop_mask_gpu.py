"""The pretrain phase's observation-token drop drawn on the device (dvla_attn_mask_obs_drop, ops.ObsDropMask,
DreamVLA.obs_drop_on_device): the kernel against the host restatement bit for bit, fresh draws under CUDA-graph replay, the
model's forward against the fp32 oracle under the drawn mask, the graphed train step against the eager one, the eager
np.random path left as it was, and train.py --cuda_graph on the LIBERO pretraining flags."""
import copy

import numpy as np
import pytest
import torch

from tests import synth
from tests.test_obs_drop_mask_cpu import ALL_HEADS, PRETRAIN_SH, restated_mask

pytestmark = pytest.mark.gpu

SMALL = dict(K=3, num_A=5, num_B=7 + 2, atten_goal=1, atten_goal_state=True, atten_only_obs=True,
             attn_robot_proprio_state=False, mask_l_obs_ratio=0.5, num_obs_token=7, action_pred_steps=2)   # L = 42


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


@pytest.fixture(autouse=True)
def keep_seed_counter(dev):
    """The tests set the process-wide dropout counter; later tests get it back as it was."""
    from dreamvla_b200 import ops
    saved = ops.seed_counter(dev).clone()
    yield
    ops.seed_counter(dev).copy_(saved)


def rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return float((a - b).norm() / (b.norm() + 1e-12))


def obs_drop_mask(kw, seed, dev):
    from dreamvla_b200 import ops
    base = restated_mask(kw, seed, 0)[0]
    n_obs = kw["num_obs_token"]
    return ops.ObsDropMask(base == 0, dev, K=kw["K"], num_A=kw["num_A"], n_obs=n_obs, n_act=kw["action_pred_steps"],
                           count=int(kw["mask_l_obs_ratio"] * n_obs), seed=seed)


def expect(kw, seed, counter, dev):
    """(packed bits, tile flags) of the restated mask at (seed, counter)."""
    from dreamvla_b200 import _lib, ops
    want = ops.AttnMask.pack_bits(restated_mask(kw, seed, counter)[1] == 0).to(dev)
    return want, _lib.attn_mask_tiles(want, want.shape[0], want.shape[0])


@pytest.mark.parametrize("kw", [PRETRAIN_SH, ALL_HEADS, SMALL], ids=["pretrain_sh", "all_heads", "small"])
def test_kernel_matches_restatement(kw, dev):
    L = kw["K"] * (kw["num_A"] + kw["num_B"])
    assert L % 32 and L % 64
    for seed in (0, 0x9E3779B97F4A7C15, (1 << 64) - 3):
        m = obs_drop_mask(kw, seed, dev)
        ctr = torch.zeros(1, dtype=torch.int64, device=dev)
        for c in (0, 1, 2, 1000003, -1):
            ctr.fill_(c)
            m.draw(ctr)
            bits, flags = expect(kw, seed, c, dev)
            assert torch.equal(m.bits, bits), (seed, c)
            assert torch.equal(m.flags, flags), (seed, c)
            assert torch.equal(m.bits | m.base_bits, m.base_bits)      # a draw only ever clears bits


def test_fresh_draws_under_captured_graph(dev):
    m = obs_drop_mask(PRETRAIN_SH, 77, dev)
    ctr = torch.zeros(1, dtype=torch.int64, device=dev)
    m.draw(ctr)                                   # first launch outside the capture
    ctr.fill_(40)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ctr.add_(1)
        m.draw(ctr)
    got = []
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        got.append((m.bits.clone(), m.flags.clone()))
    for (bits, flags), c in zip(got, (41, 42)):
        want_bits, want_flags = expect(PRETRAIN_SH, 77, c, dev)
        assert torch.equal(bits, want_bits) and torch.equal(flags, want_flags), c
    assert not torch.equal(got[0][0], got[1][0])


def pretrain_model(dev, layers=2):
    """synth's pretrain_mlp model in the pretrain phase with the LIBERO pretraining drop ratio, dropout off."""
    from dreamvla_b200.models import DreamVLA
    cfg = dict(synth.CASES["pretrain_mlp"], phase="pretrain", mask_l_obs_ratio=0.5, transformer_layers=layers)
    torch.manual_seed(0)
    m = DreamVLA(finetune_type="calvin", clip_device="cpu", vit_checkpoint_path=None, **synth.ctor_kwargs(cfg))
    sd = synth.synth_state_dict(m.state_dict(), cfg["weight_seed"])
    m.load_state_dict(sd)
    m = m.bfloat16().to(dev)
    m._init_model_type()
    m.train()
    gp = m.transformer_backbone
    gp.embd_pdrop = 0.0
    for blk in gp.h:
        blk.attn.attn_pdrop = blk.attn.resid_pdrop = blk.mlp.resid_pdrop = 0.0
    kw = dict(K=cfg["sequence_length"], num_A=36, num_B=18 + 3, atten_goal=cfg["atten_goal"],
              atten_goal_state=cfg["atten_goal_state"], atten_only_obs=True,
              attn_robot_proprio_state=cfg["attn_robot_proprio_state"], mask_l_obs_ratio=0.5, num_obs_token=18,
              action_pred_steps=3)
    return m, sd, cfg, kw


def test_forward_matches_oracle_under_the_drawn_mask(dev):
    from dreamvla_b200 import ops
    from oracle import dreamvla_oracle as O
    m, sd, cfg, kw = pretrain_model(dev)
    assert m.redraws_mask and not m.obs_drop_on_device
    torch.manual_seed(3)
    m.obs_drop_on_device = True
    ops.seed_counter(dev).fill_(5)
    inp = synth.synth_inputs(cfg)
    with torch.no_grad():
        out = m(*(inp[k].to(dev) for k in ("image_primary", "image_wrist", "state", "text_token")),
                action_label=inp["action_label"].to(dev))
    base, want, _ = restated_mask(kw, m._obs_drop_mask.seed, 5)
    assert torch.equal(m._obs_drop_mask.bits, ops.AttnMask.pack_bits(want == 0).to(dev))
    got = torch.cat([out[0].flatten(), out[1].flatten()])
    ref = {}
    for name, mask in (("drawn", want), ("no drop", base)):
        with torch.no_grad():
            o = O.dreamvla_forward(dict(sd, attention_mask=mask), cfg, inp["image_primary"], inp["image_wrist"],
                                   inp["state"], inp["text_token"], action_label=inp["action_label"])
        ref[name] = torch.cat([o["arm_pred_action"].flatten(), o["gripper_pred_action"].flatten()])
    e_drawn, e_base = rel(got, ref["drawn"]), rel(got, ref["no drop"])
    print(f"arm+gripper rel-L2 vs the oracle: {e_drawn:.2e} under the drawn mask, {e_base:.2e} without the drop")
    assert e_drawn < 2e-2
    assert e_base > 2e-2


def test_graphed_step_matches_eager_device_draw(dev):
    from dreamvla_b200 import ops
    from dreamvla_b200.utils.train_utils import GraphedTrainStep, StepConfig, TrainStep, synthetic_batch
    m1, _, cfg, kw = pretrain_model(dev)
    m2 = copy.deepcopy(m1)
    scfg = StepConfig(sequence_length=cfg["sequence_length"], use_dit_head=False, loss_action=True, loss_image=True,
                      atten_goal=cfg["atten_goal"], learning_rate=1e-4, weight_decay=1e-2, gradient_accumulation_steps=2,
                      reduce_every_micro_step=True)
    batch = synthetic_batch(scfg, 1, dev, seed=9)
    ctr = ops.seed_counter(dev)

    torch.manual_seed(123)
    ctr.zero_()
    graphed = GraphedTrainStep(TrainStep(m1, scfg), batch, warmup=2)       # 2 real warm-up micro-steps
    assert m1.obs_drop_on_device
    losses_g, bits_g = [], []
    for _ in range(4):
        losses_g.append(float(graphed(batch)))
        bits_g.append(m1._obs_drop_mask.bits.clone())
    assert int(ctr) == 6

    torch.manual_seed(123)
    ctr.zero_()
    eager = TrainStep(m2, scfg)
    m2.obs_drop_on_device = True
    assert m2._obs_drop_mask.seed == m1._obs_drop_mask.seed
    losses_e, bits_e = [], []
    for _ in range(6):
        losses_e.append(float(eager(batch)))
        bits_e.append(m2._obs_drop_mask.bits.clone())
    for i, (a, b) in enumerate(zip(losses_e[2:], losses_g)):
        tol = 2e-2 if i == 0 else 8e-2
        assert abs(a - b) < tol * abs(a) + 1e-4, (losses_e, losses_g)
    for i, (a, b) in enumerate(zip(bits_e[2:], bits_g)):
        assert torch.equal(a, b), i
        assert torch.equal(a, expect(kw, m1._obs_drop_mask.seed, 3 + i, dev)[0]), i
    assert not torch.equal(bits_g[0], bits_g[1])


def test_eager_model_draws_through_numpy(dev, monkeypatch):
    """A model never switched to the device draw keeps the reference's call sequence: K np.random.choice calls per training
    forward, and the mask parameter is replaced by the one they produced."""
    m, _, cfg, kw = pretrain_model(dev)
    calls = []
    choice = np.random.choice

    def counting(*a, **k):
        calls.append(k.get("size"))
        return choice(*a, **k)

    monkeypatch.setattr(np.random, "choice", counting)
    inp = synth.synth_inputs(cfg)
    for n in (1, 2):
        np.random.seed(11)
        with torch.no_grad():
            m(*(inp[k].to(dev) for k in ("image_primary", "image_wrist", "state", "text_token")),
              action_label=inp["action_label"].to(dev))
        assert calls == [9] * (kw["K"] * n)
        assert not m.obs_drop_on_device and m._obs_drop_mask is None
    np.random.seed(11)
    from dreamvla_b200.models.dreamvla_model import generate_attention_mask
    assert torch.equal(m.attention_mask.float().cpu(), generate_attention_mask(**kw))


PRETRAIN_FLAGS = ["--traj_cons", "--rgb_pad", "10", "--gripper_pad", "4", "--bf16_module", "vision_encoder", "--seed", "42",
                  "--batch_size", "10", "--precision", "fp32", "--learning_rate", "1e-4", "--finetune_type", "libero_pretrain",
                  "--weight_decay", "1e-4", "--lr_scheduler", "cosine", "--warmup_epochs", "1", "--num_resampler_query", "16",
                  "--num_obs_token_per_image", "9", "--transformer_layers", "2", "--hidden_dim", "1024",
                  "--transformer_heads", "16", "--phase", "pretrain", "--obs_pred", "--sequence_length", "11",
                  "--action_pred_steps", "3", "--future_steps", "3", "--atten_goal", "4", "--window_size", "11",
                  "--loss_image", "--loss_action", "--gripper_width", "--atten_only_obs", "--atten_goal_state",
                  "--mask_l_obs_ratio", "0.5", "--attn_robot_proprio_state", "--attn_implementation", "sdpa"]


def test_train_py_captures_the_libero_pretrain_recipe(dev):
    """scripts/LIBERO/DreamVLA/pretrain.sh's flags (2 layers) with --cuda_graph: one eager micro-step, then the captured step
    replays with the device draw; every loss stays finite."""
    import train
    from dreamvla_b200.utils.arguments_utils import get_parser
    args = get_parser().parse_args(PRETRAIN_FLAGS + ["--synthetic_steps", "5", "--gradient_accumulation_steps", "2",
                                                     "--cuda_graph"])
    state = train.main(args)
    assert state.total_micro == 5 and float(state.flat.step_count) == 3.0
    assert getattr(state.model, "_dvla_graphed_step", None) is not None, "--cuda_graph did not capture"
    assert state.model.obs_drop_on_device
    assert all(torch.isfinite(v).all() for v in state.last_terms.values())
    assert torch.isfinite(state.model._dvla_graphed_step.loss).all()
