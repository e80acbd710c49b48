"""CLIP's image transform on the device (dvla_image_fn, `data_utils.preprocess_image`): bit-identical to torchvision + Pillow
on the golden crops (tests/golden/image_fn.pt) in fp32 and bf16, batches and vertical flips, argument errors; and through the
layers above it: a train step on raw uint8 frames sees exactly the image tensors and loss of host-preprocessed ones,
`train.main` trains from a raw-frame loader with --cuda_graph --device_augment, and the CALVIN / LIBERO rollout wrappers
return the same actions from raw frames as from host-preprocessed tensors."""
import ctypes
import importlib.util
import os

import numpy as np
import pytest
import torch

from tests import synth

pytestmark = pytest.mark.gpu

_spec = importlib.util.spec_from_file_location(
    "make_golden_image_fn", os.path.join(os.path.dirname(__file__), "golden", "make_golden_image_fn.py"))
G = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(G)


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def through_lut(crop_hwc, lut):
    """uint8 [..., 224, 224, 3] crop -> ToTensor + Normalize as the [3, 256] table gives it: fp32 [..., 3, 224, 224]."""
    idx = crop_hwc.long().movedim(-1, -3)
    return torch.stack([lut[c][idx[..., c, :, :]] for c in range(3)], dim=-3)


def host_image_fn(frame_hwc):
    """The reference's `image_processor` on the host: CLIP `_transform(224)` through torchvision + Pillow -> fp32 [3, 224, 224]."""
    from PIL import Image
    import torchvision.transforms as T
    from dreamvla_b200.utils.data_utils import CLIP_MEAN, CLIP_STD
    tf = T.Compose([T.Resize(224, interpolation=T.InterpolationMode.BICUBIC), T.CenterCrop(224), T.ToTensor(),
                    T.Normalize(CLIP_MEAN, CLIP_STD)])
    return tf(Image.fromarray(np.ascontiguousarray(np.asarray(frame_hwc))).convert("RGB"))


def test_kernel_matches_golden_crops(dev):
    from dreamvla_b200.utils.data_utils import image_fn_lut, preprocess_image
    crops, gold = G.load_crops()
    lut = image_fn_lut("cpu")
    for name, frame in G.make_inputs(gold["seed"], gold["shapes"]):
        want = through_lut(crops[name], lut)
        got = preprocess_image(frame.to(dev)).cpu()
        assert got.shape == (3, 224, 224) and got.dtype == torch.float32
        assert torch.equal(got, want), (name, int((got != want).sum()))
        got16 = preprocess_image(frame.to(dev), torch.bfloat16).cpu()
        assert torch.equal(got16, want.to(torch.bfloat16)), name


def test_batches_and_vertical_flip(dev):
    from dreamvla_b200.utils.data_utils import preprocess_image
    for h, w in ((200, 200), (84, 84), (128, 128), (480, 640), (7, 5)):
        g = torch.Generator().manual_seed(h * 1000 + w)
        frames = torch.randint(0, 256, (2, 3, h, w, 3), generator=g, dtype=torch.uint8).to(dev)
        batch = preprocess_image(frames)
        assert batch.shape == (2, 3, 3, 224, 224)
        for i in range(2):
            for j in range(3):
                assert torch.equal(batch[i, j], preprocess_image(frames[i, j])), (h, w, i, j)
        flipped = preprocess_image(frames, torch.bfloat16, flip_vertical=True)
        assert torch.equal(flipped, preprocess_image(frames.flip(2).contiguous(), torch.bfloat16)), (h, w)
    # LIBERO's agent view: the reference flips the frame (obs[...][::-1]) before Pillow
    frame = torch.randint(0, 256, (128, 128, 3), generator=torch.Generator().manual_seed(8), dtype=torch.uint8)
    assert torch.equal(preprocess_image(frame.to(dev), flip_vertical=True).cpu(), host_image_fn(frame.numpy()[::-1]))


def test_invalid_arguments_never_launch(dev):
    from dreamvla_b200 import _lib as L
    from dreamvla_b200.utils.data_utils import image_fn_lut
    lib = L.load()
    frames = torch.zeros(2, 200, 200, 3, dtype=torch.uint8, device=dev)
    out = torch.empty(2, 3, 224, 224, device=dev)
    xb, xc, yb, yc = L.image_fn_tables(200, 200, dev)
    lut = image_fn_lut(dev)

    def args(**kw):
        a = L.ImageFnArgs(frames.data_ptr(), out.data_ptr(), 2, 200, 200, 3, xb.data_ptr(), xc.data_ptr(), yb.data_ptr(),
                          yc.data_ptr(), lut.data_ptr(), 0, 0)
        for k, v in kw.items():
            setattr(a, k, v)
        return a
    stream = L._stream()
    assert lib.dvla_image_fn(ctypes.byref(args()), stream) == 0
    torch.cuda.synchronize()
    bad = [dict(frames=None), dict(out=None), dict(xcoeffs=None), dict(ybounds=None), dict(lut=None), dict(c=4), dict(c=1),
           dict(h=0), dict(w=-3), dict(h=3585), dict(w=100000), dict(n=-1), dict(out_dtype=2), dict(out_dtype=-1),
           dict(out=out.data_ptr() + 4)]
    n0 = L.launch_count()
    for kw in bad:
        assert lib.dvla_image_fn(ctypes.byref(args(**kw)), stream) == -1, kw
        assert b"image_fn" in lib.dvla_last_error(), kw
    assert lib.dvla_image_fn(None, stream) == -1
    assert lib.dvla_image_fn(ctypes.byref(args(n=0, frames=None, out=None)), stream) == 0, "an empty batch is a no-op"
    assert L.launch_count() == n0, "no launch on invalid or empty input"
    empty = L.image_fn(torch.empty(0, 50, 60, 3, dtype=torch.uint8, device=dev), lut)
    assert empty.shape == (0, 3, 224, 224)
    with pytest.raises(RuntimeError, match="3 channels"):
        L.image_fn(torch.zeros(1, 50, 60, 4, dtype=torch.uint8, device=dev), lut)
    torch.cuda.synchronize()


# ---- train step --------------------------------------------------------------------------------------------------------------
def raw_and_host_windows(B, W, seed):
    """uint8 [B, W, 200, 200, 3] / [B, W, 84, 84, 3] camera windows and their host-preprocessed fp32 [B, W, 3, 224, 224]."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for key, side in (("images_primary", 200), ("images_wrist", 84)):
        raw = torch.randint(0, 256, (B, W, side, side, 3), generator=g, dtype=torch.uint8)
        host = torch.stack([torch.stack([host_image_fn(raw[b, t].numpy()) for t in range(W)]) for b in range(B)])
        out[key] = (raw, host)
    return out


def test_train_step_on_raw_frames_matches_host_preprocessing(dev):
    from dreamvla_b200.models import DreamVLA
    from dreamvla_b200.utils.data_utils import prepare_batch
    from dreamvla_b200.utils.train_utils import StepConfig, TrainStep, synthetic_batch
    cfg = synth.CASES["libero_dit"]
    torch.manual_seed(0)
    m = DreamVLA(finetune_type="calvin", clip_device="cpu", vit_checkpoint_path=None, **synth.ctor_kwargs(cfg))
    m.load_state_dict(synth.synth_state_dict(m.state_dict(), cfg["weight_seed"]))
    m = m.bfloat16().to(dev)
    m._init_model_type()
    m.train()
    m.transformer_backbone.embd_pdrop = 0.0
    for blk in m.transformer_backbone.h:
        blk.attn.attn_pdrop = blk.attn.resid_pdrop = blk.mlp.resid_pdrop = 0.0
    scfg = StepConfig(sequence_length=cfg["sequence_length"], use_dit_head=True, learning_rate=1e-5)
    step = TrainStep(m, scfg)
    B, W = 2, scfg.sequence_length + scfg.future_steps
    base = synthetic_batch(scfg, B, dev, seed=3)
    wins = raw_and_host_windows(B, W, seed=5)
    host = dict(base, **{k: h.to(dev).to(torch.bfloat16) for k, (_, h) in wins.items()})      # prefetch_to_device's cast
    raw = prepare_batch(dict(base, **{k: r.to(dev) for k, (r, _) in wins.items()}))
    for k in wins:
        assert raw[k].dtype == torch.bfloat16 and torch.equal(raw[k], host[k]), k
    g = torch.Generator().manual_seed(6)
    n = 8 * B * scfg.sequence_length
    draws = dict(diffusion_noise=torch.randn(n, 3, 7, generator=g).to(dev),
                 diffusion_timestep=torch.randint(0, 100, (n,), generator=g).to(dev),
                 diffusion_drop_ids=(torch.rand(n, generator=g) < 0.1).long().to(dev))
    l_host = step.forward_backward(host, draws)
    l_raw = step.forward_backward(raw, draws)
    step.flat.G.zero_()
    assert torch.isfinite(l_host) and torch.equal(l_host, l_raw), (float(l_host), float(l_raw))


def test_train_main_with_raw_frame_loader(dev):
    import train
    from dreamvla_b200.utils.arguments_utils import get_parser
    from dreamvla_b200.utils.train_utils import StepConfig, synthetic_batch
    from tests.test_train_entry_gpu import FLAGS
    args = get_parser().parse_args(FLAGS + ["--cuda_graph", "--device_augment", "--rgb_pad", "10", "--gripper_pad", "4"])

    class RawLoader:
        num_batches = 4

        def __iter__(self):
            cfg = StepConfig.from_args(args)
            W = cfg.sequence_length + cfg.future_steps
            for i in range(self.num_batches):
                b = synthetic_batch(cfg, args.batch_size, "cpu", seed=100 + i, dtype=torch.float32)
                g = torch.Generator().manual_seed(i)
                prim = torch.randint(0, 256, (args.batch_size, W, 200, 200, 3), generator=g, dtype=torch.uint8)
                wrist = torch.randint(0, 256, (args.batch_size, W, 84, 84, 3), generator=g, dtype=torch.uint8)
                yield (prim, b["text"], b["actions"], wrist, b["states"], None, None, None, None, None, None, None, {})

    state = train.main(args, RawLoader())
    assert state.total_micro == 4 and float(state.flat.step_count) == 4.0
    graphed = getattr(state.model, "_dvla_graphed_step", None)
    assert graphed is not None and graphed.static["images_primary"].shape[-3:] == (3, 224, 224)
    assert graphed.static["images_primary"].dtype == torch.bfloat16
    assert all(torch.isfinite(v).all() for v in state.last_terms.values())
    args.device_augment = False
    with pytest.raises(ValueError, match="--device_augment"):
        train.main(args, RawLoader())


# ---- rollouts ----------------------------------------------------------------------------------------------------------------
def rollout_model(dev):
    from dreamvla_b200.models import DreamVLA
    cfg = synth.CASES["libero_dit"]
    torch.manual_seed(0)
    m = DreamVLA(finetune_type="calvin", clip_device="cpu", vit_checkpoint_path=None, **synth.ctor_kwargs(cfg))
    m.load_state_dict(synth.synth_state_dict(m.state_dict(), cfg["weight_seed"]))
    m = m.bfloat16().to(dev)
    m._init_model_type()
    # the fused one-sequence sampler adds split-K partial sums with fp32 atomics (run-to-run order); the module sampler is
    # deterministic, so two wrappers fed the same images return the same actions bit for bit
    m.FUSED_SAMPLER = False
    return m.eval(), cfg["sequence_length"]


@pytest.mark.parametrize("incremental,graph", [(False, False), (False, True), (True, True)])
def test_calvin_wrapper_raw_frames_match_preprocessed(dev, incremental, graph):
    from dreamvla_b200.utils.eval_utils_calvin import ModelWrapper
    model, S = rollout_model(dev)
    kw = dict(history_len=S, device=dev, use_cuda_graph=graph, incremental=incremental, prune=False)
    w_host, w_raw = ModelWrapper(model, **kw), ModelWrapper(model, **kw)
    g = torch.Generator().manual_seed(31)
    text = torch.zeros(77, dtype=torch.long)
    text[0], text[1:6], text[6] = 49406, torch.randint(1, 49406, (5,), generator=g), 49407
    for i in range(S + 2):
        static = torch.randint(0, 256, (200, 200, 3), generator=g, dtype=torch.uint8).numpy()
        grip = torch.randint(0, 256, (84, 84, 3), generator=g, dtype=torch.uint8).numpy()
        obs = torch.randn(15, generator=g) * 0.5
        noise = torch.randn(S, 3, 7, generator=g)
        a = w_host.step(host_image_fn(static), host_image_fn(grip), obs, text, sample_noise=noise)
        b = w_raw.step(static, torch.from_numpy(grip), obs, text, sample_noise=noise)
        assert np.array_equal(a, b), (i, a, b)


@pytest.mark.parametrize("incremental", [False, True])
def test_libero_wrapper_flips_raw_agent_view(dev, incremental):
    from dreamvla_b200.utils.eval_utils_libero import ModelWrapper
    model, S = rollout_model(dev)
    kw = dict(history_len=S, device=dev, use_cuda_graph=True, incremental=incremental, prune=False)
    w_host, w_raw = ModelWrapper(model, **kw), ModelWrapper(model, **kw)
    g = torch.Generator().manual_seed(41)
    text = torch.zeros(77, dtype=torch.long)
    text[0], text[1:4], text[4] = 49406, torch.randint(1, 49406, (3,), generator=g), 49407
    for t in range(S + 2):
        agent = torch.randint(0, 256, (128, 128, 3), generator=g, dtype=torch.uint8).numpy()
        hand = torch.randint(0, 256, (128, 128, 3), generator=g, dtype=torch.uint8).numpy()
        pos, quat = torch.randn(3, generator=g).numpy() * 0.3, torch.randn(4, generator=g).numpy()
        noise = torch.randn(S, 3, 7, generator=g)
        a = w_host.step(host_image_fn(agent[::-1]), host_image_fn(hand), pos, quat, None, text, t, sample_noise=noise)
        b = w_raw.step(agent, hand, pos, quat, None, text, t, sample_noise=noise)
        assert np.array_equal(a, b), (t, a, b)
