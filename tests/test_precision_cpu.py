"""`--precision fp32` (fp32 master weights, bf16 working copy) without a GPU: the precision rules of train.py, the exported
fp32-master AdamW entry point, and its register budget on sm_90a."""
import ctypes
import os
import re
import subprocess
import types

import pytest

from dreamvla_b200 import build

# the flags of the reference's scripts/CALVIN_ABC_D/DreamVLA/finetune.sh (paths replaced by placeholders)
FINETUNE_SH = [
    "--traj_cons", "--rgb_pad", "10", "--gripper_pad", "4", "--gradient_accumulation_steps", "1",
    "--bf16_module", "vision_encoder", "--vit_checkpoint_path", "vit.pth", "--calvin_dataset", "data/", "--workers", "16",
    "--lr_scheduler", "cosine", "--save_every_iter", "100000", "--num_epochs", "20", "--seed", "42", "--batch_size", "2",
    "--precision", "fp32", "--learning_rate", "1e-3", "--finetune_type", "calvin", "--wandb_project", "p",
    "--weight_decay", "1e-4", "--num_resampler_query", "16", "--num_obs_token_per_image", "9", "--run_name", "r",
    "--save_checkpoint", "--save_checkpoint_path", "ck/", "--transformer_layers", "24", "--hidden_dim", "1024",
    "--transformer_heads", "16", "--phase", "finetune", "--action_pred_steps", "3", "--sequence_length", "10",
    "--future_steps", "3", "--window_size", "13", "--obs_pred", "--depth_pred", "--use_dit_head", "--loss_image",
    "--loss_action", "--loss_depth", "--track_label_patch_size", "8", "--load_track_labels", "--track_label_path", "t/",
    "--loss_sam_feat", "--sam_feat_pred", "--load_sam_features", "--sam_feature_path", "s/", "--flow_as_mask",
    "--attn_implementation", "sdpa", "--reset_obs_token", "--reset_action_decoder", "--report_to_wandb",
    "--finetune_from_pretrained_ckpt", "pre.pth",
]


def ns(precision, bf16_module=""):
    return types.SimpleNamespace(precision=precision, bf16_module=bf16_module)


def test_resolve_precision_rules():
    from train import resolve_precision
    for p in ("bf16", "amp_bf16", "amp_bfloat16"):
        assert resolve_precision(ns(p)) == "bf16"
        assert resolve_precision(ns(p, "causal_transformer")) == "bf16"          # bf16 mode: everything is bf16 anyway
    for spec in ("", "vision_encoder", "text_encoder", "vision_encoder,text_encoder", "vision_encoder text_encoder"):
        assert resolve_precision(ns("fp32", spec)) == "fp32", spec
    for spec in ("causal_transformer", "perceiver_resampler", "vision_encoder,causal_transformer", "action_decoder",
                 "image_primary_projector", "sam_decoder"):
        with pytest.raises(SystemExit, match="trained modules"):
            resolve_precision(ns("fp32", spec))
    with pytest.raises(SystemExit, match="unknown module"):
        resolve_precision(ns("fp32", "vision_encodr"))
    for p in ("fp16", "bf16_and_fp32"):
        with pytest.raises(SystemExit, match="not supported"):
            resolve_precision(ns(p, "vision_encoder"))


def test_reference_finetune_flags_resolve_to_fp32():
    from dreamvla_b200.utils.arguments_utils import get_parser
    from train import resolve_precision
    args = get_parser().parse_args(FINETUNE_SH)
    assert args.precision == "fp32" and args.bf16_module == "vision_encoder"
    assert resolve_precision(args) == "fp32"
    assert resolve_precision(get_parser().parse_args([])) == "fp32"                # the reference's default precision


def test_adamw_master_declared_and_exported(repo_root):
    header = open(os.path.join(repo_root, "include", "dvla.h")).read()
    assert re.search(r"int\s+dvla_adamw_master\s*\(\s*const\s+dvla_adamw_master_args\s*\*", header)
    lib = ctypes.CDLL(build.build_library())
    assert hasattr(lib, "dvla_adamw_master")


def test_adamw_master_kernel_does_not_spill(tmp_path):
    src = os.path.join(build.CSRC, "loss_optim.cu")
    cmd = [build._nvcc(), *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "loss_optim.o")]
    try:
        r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    except FileNotFoundError:
        pytest.skip("nvcc not available")
    assert r.returncode == 0, r.stderr
    # ptxas prints "Compiling entry function '<mangled>'", then its properties (stack frame, spills) and register count
    blocks = re.split(r"Compiling entry function", r.stderr)
    mine = [b for b in blocks if "adamw_master_kernel" in b.split("\n", 1)[0]]
    assert len(mine) == 1, r.stderr
    m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", mine[0])
    assert m is not None, mine[0]
    assert (int(m.group(1)), int(m.group(2))) == (0, 0), mine[0]
