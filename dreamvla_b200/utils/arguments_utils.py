"""Command-line flags of the entry points -- accepts every flag of reference utils/arguments_utils.py:43-308 with the
same names, types and defaults (table-driven; the reference's data-loading flags are parsed and ignored by the hot path).
"""
from __future__ import annotations

import argparse

# (flag, type or "flag" for store_true, default[, choices])
_FLAGS = [
    ("--run_name", str, "RobotFlamingo"), ("--offline", "flag", False), ("--num_epochs", int, 1), ("--batch_size", int, 1),
    ("--gradient_accumulation_steps", int, 1), ("--resume_from_checkpoint", str, None),
    ("--delete_previous_checkpoint", "flag", False), ("--seed", int, 42), ("--learning_rate", float, 1e-4),
    ("--lr_scheduler", str, "constant"), ("--calvin_dataset", str, ""), ("--warmup_epochs", int, 1), ("--local-rank", int, 0),
    ("--weight_decay", float, 0.1),
    ("--precision", str, "fp32", ["amp_bf16", "amp_bfloat16", "bf16", "fp16", "fp32", "bf16_and_fp32"]),
    ("--pred_num", int, 1), ("--workers", int, 16), ("--dist-url", str, "env://"), ("--dist-backend", str, "nccl"),
    ("--no-set-device-rank", "flag", False), ("--report_to_wandb", "flag", False), ("--wandb_project", str, None),
    ("--wandb_entity", str, None), ("--save_checkpoints_to_wandb", "flag", False), ("--rgb_pad", int, -1),
    ("--gripper_pad", int, -1), ("--traj_cons", "flag", False), ("--text_aug", "flag", False), ("--residual", "flag", False),
    ("--dif_ws", "flag", False), ("--partial_data", "flag", False), ("--save_every_iter", int, -1),
    ("--min_window_size", int, 12), ("--max_window_size", int, 24), ("--multi_step_action", int, 1),
    ("--data_in_ceph", "flag", False), ("--root_dir", str, "s3://real_data"), ("--image_primary_size", int, 200),
    ("--image_wrist_size", int, 84), ("--finetune_type", str, ""), ("--start_save_checkpoint", int, -1),
    ("--save_checkpoint", "flag", False), ("--save_checkpoint_path", str, "./checkpoints/"), ("--save_checkpoint_seq", int, 1),
    ("--validation", "flag", False), ("--bf16_module", str, ""), ("--sequence_length", int, 10), ("--future_steps", int, 3),
    ("--num_resampler_query", int, 9), ("--num_obs_token_per_image", int, 9), ("--calvin_input_image_size", int, 224),
    ("--patch_size", int, 16), ("--primary_mode", str, "image_primary"), ("--small_size", int, 0),
    ("--dataset_info", str, "droid_success"), ("--finetune_from_pretrained_ckpt", str, None),
    ("--loss_arm_action_ratio", float, 1.0), ("--loss_gripper_action_ratio", float, 0.01), ("--action_pred_steps", int, 1),
    ("--dit_type", str, "DiT-B"), ("--obs_pred", "flag", False), ("--atten_only_obs", "flag", False),
    ("--attn_robot_proprio_state", "flag", False), ("--atten_goal", int, 0), ("--atten_goal_state", "flag", False),
    ("--use_dinosiglip", "flag", False), ("--use_dit_head", "flag", False), ("--use_fm", "flag", False),
    ("--depth_pred", "flag", False), ("--use_depth_query", "flag", False), ("--use_dpt_head", "flag", False),
    ("--dino_feat_pred", "flag", False), ("--sam_feat_pred", "flag", False), ("--trajectory_pred", "flag", False),
    ("--use_trajectory_query", "flag", False), ("--track_label_patch_size", int, 8), ("--no_pred_gripper_traj", "flag", False),
    ("--no_unshuffle", "flag", False), ("--flow_as_mask", "flag", False), ("--share_query", "flag", False),
    ("--attn_implementation", str, "eager"), ("--use_gpt2_pretrained", "flag", False), ("--mask_l_obs_ratio", float, 0.0),
    ("--reset_action_token", "flag", False), ("--reset_obs_token", "flag", False), ("--reset_mask_token", "flag", False),
    ("--reset_image_decoder", "flag", False), ("--reset_action_decoder", "flag", False), ("--reset_resampler", "flag", False),
    ("--loss_action", "flag", False), ("--loss_image", "flag", False), ("--loss_depth", "flag", False),
    ("--loss_dino_feat", "flag", False), ("--loss_sam_feat", "flag", False), ("--loss_trajectory", "flag", False),
    ("--except_lang", "flag", False), ("--load_track_labels", "flag", False), ("--track_label_path", str, None),
    ("--load_dino_features", "flag", False), ("--dino_features_path", str, None), ("--load_sam_features", "flag", False),
    ("--sam_features_path", str, None), ("--sam_feature_path", str, None), ("--dino_feature_path", str, None),
    ("--merge_data", "flag", False), ("--transformer_layers", int, 12),
    ("--hidden_dim", int, 384), ("--transformer_heads", int, 12), ("--phase", str, "finetune"),
    ("--libero_path", str, ""), ("--libero_img_size", int, 128), ("--libero_eval_max_steps", int, 600),
    ("--gripper_width", "flag", False), ("--load_libero_file", str, "h5"), ("--eval_libero_ensembling", "flag", False),
    ("--ensembling_temp", float, 0.01), ("--real_dataset_names", str, None), ("--use_aug_data", "flag", False),
    ("--real_eval_max_steps", int, 600), ("--max_rel_pos", float, 0.02), ("--max_rel_orn", float, 0.05),
    ("--magic_scaling_factor_pos", float, 1.0), ("--magic_scaling_factor_orn", float, 1.0), ("--calvin_conf_path", str, None),
    ("--future_act_len", int, -1), ("--visualize", "flag", False), ("--reset", "flag", False), ("--diverse_inst", "flag", False),
    ("--pad_length", int, -1), ("--window_size", int, 13), ("--vit_checkpoint_path", str, None),
]
# added by this repo (not in the reference)
# --device_augment: apply the collator's RandomShiftsAug (--rgb_pad / --gripper_pad / --traj_cons, reference
# utils/data_utils.py:1337-1354) on the GPU to the transferred batch (utils/data_utils.py here); the loader must then be built
# WITHOUT pads so that the augmentation is not applied twice.  A loader may ship raw uint8 camera frames instead of
# preprocessed ones (no flag: the dtype decides); CLIP's image transform then runs on the device before the shifts.
# --exchange_on_boundary_only: with gradient accumulation, all-reduce + clip once per optimiser step instead of the
# reference's every-micro-step exchange and in-place clip (utils/train_utils.py:599-600); a different update, opt-in.
_EXTRA = [("--synthetic_steps", int, 0), ("--cuda_graph", "flag", False), ("--synthetic_rollout_steps", int, 0),
          ("--exchange_on_boundary_only", "flag", False), ("--incremental_rollout", "flag", False), ("--num_envs", int, 1),
          ("--device_augment", "flag", False)]


def get_parser() -> argparse.ArgumentParser:
    parser = argparse.ArgumentParser(description="DreamVLA hot path on H100 (reference-compatible flags)")
    for spec in _FLAGS + _EXTRA:
        name, typ, default = spec[0], spec[1], spec[2]
        if typ == "flag":
            parser.add_argument(name, default=default, action="store_true")
        elif len(spec) > 3:
            parser.add_argument(name, type=typ, default=default, choices=spec[3])
        else:
            parser.add_argument(name, type=typ, default=default)
    return parser


MODEL_KWARGS = ("sequence_length", "num_resampler_query", "num_obs_token_per_image", "calvin_input_image_size", "patch_size",
                "action_pred_steps", "obs_pred", "atten_only_obs", "attn_robot_proprio_state", "atten_goal",
                "atten_goal_state", "mask_l_obs_ratio", "transformer_layers", "hidden_dim", "transformer_heads", "phase",
                "gripper_width", "pred_num", "depth_pred", "trajectory_pred", "use_depth_query", "use_dpt_head",
                "use_trajectory_query", "track_label_patch_size", "dino_feat_pred", "sam_feat_pred", "use_dinosiglip",
                "use_dit_head", "use_gpt2_pretrained", "no_pred_gripper_traj", "no_unshuffle", "share_query",
                "attn_implementation", "use_fm", "dit_type")


def model_kwargs(args) -> dict:
    """The ctor kwargs train.py:55-97 passes from the flags."""
    return {k: getattr(args, k) for k in MODEL_KWARGS}
