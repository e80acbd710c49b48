"""ncu driver: a few attention launches at the path's per-GPU-batch-8 shapes ."""
import sys

import torch

sys.path.insert(0, __file__.rsplit("/tools/", 1)[0])
from dreamvla_b200 import _lib as L  # noqa: E402

dev = "cuda"
what = sys.argv[1] if len(sys.argv) > 1 else "dec"
B, H, Lq = {"dec": (160, 16, 265), "vit": (160, 12, 197), "gpt": (8, 16, 1290)}[what]
qkv = torch.randn(B, Lq, 3, H, 64, device=dev, dtype=torch.bfloat16)
q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
bits = flags = None
p_drop = 0.0
if what == "gpt":      # the backbone's real block mask (dreamvla_model.py:25-66) and attn_pdrop
    from dreamvla_b200 import ops
    from dreamvla_b200.models.dreamvla_model import generate_attention_mask
    add = generate_attention_mask(K=10, num_A=36, num_B=93, atten_goal=0, atten_goal_state=False, atten_only_obs=False,
                                  attn_robot_proprio_state=False, mask_l_obs_ratio=0.0, num_obs_token=90, action_pred_steps=3)
    am = ops.AttnMask(add == 0, dev)
    bits, flags = am.bits, am.flags
    p_drop = 0.1
for _ in range(3):
    o, lse = L.attn_fwd(q, k, v, 0.125, bits, flags, dropout_p=p_drop, dropout_seed=5)
if len(sys.argv) > 2 and sys.argv[2] == "bwd":
    d_o = torch.randn_like(o)
    dqkv = torch.empty_like(qkv)
    for _ in range(2):
        L.attn_bwd(q, k, v, o, d_o, lse, 0.125, dqkv[:, :, 0], dqkv[:, :, 1], dqkv[:, :, 2], bits, flags,
                   dropout_p=p_drop, dropout_seed=5)
torch.cuda.synchronize()
