"""TEST INFRASTRUCTURE (never imported by dreamvla_b200/): CPU restatement of the two device-side collator pieces of SURVEY.md
8f-2 -- the reference's `RandomShiftsAug` (utils/data_utils.py:326-383) and the NEAREST depth resize of `depth_image_fn`
(utils/data_utils.py:3588-3603) -- pinned against the reference's own code by tests/test_augment_cpu.py (through the reference
outputs recorded in tests/golden/augment.pt and tests/golden/reference_checks.pt).

Two forms of the augmentation are given:
  * `random_shifts_grid_sample` follows the reference line by line: replicate pad, fp32 grid of the padded image's pixel
    centres, integer shift * 2/(h+2*pad), `F.grid_sample(bilinear, zeros, align_corners=False)`;
  * `shift_crop` is the closed form the CUDA kernel computes (include/dvla.h `dvla_shift_crop`): a crop of the replicate-padded
    image at an integer offset, i.e. clamped indexing.  The two differ only by the fp32 rounding of the grid coordinates
    (bilinear weights (1-e, e) with e ~ 1e-5 instead of (1, 0)); the test bounds that difference.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F


def draw_shifts(n, pad, low, generator=None, dtype=torch.float32):
    """The reference's draw (data_utils.py:345-349 `forward`: low = 0; :372-376 `forward_traj`: low = 1): torch.randint(low,
    2*pad+1, (n, 1, 1, 2)) in the image dtype; returned as the integer (sx, sy) pairs [n, 2]."""
    s = torch.randint(low, 2 * pad + 1, size=(n, 1, 1, 2), dtype=dtype, generator=generator)
    return s.view(n, 2).to(torch.int32)


def random_shifts_grid_sample(x, shifts_xy, pad):
    """data_utils.py:330-354 with the shift passed in: x [n, c, h, w] float, shifts_xy int [n, 2] = (sx, sy)."""
    n, c, h, w = x.size()
    assert h == w
    xp = F.pad(x, (pad,) * 4, "replicate")                                            # :333-334
    eps = 1.0 / (h + 2 * pad)                                                           # :335
    arange = torch.linspace(-1.0 + eps, 1.0 - eps, h + 2 * pad, dtype=x.dtype)[:h]      # :336-340
    arange = arange.unsqueeze(0).repeat(h, 1).unsqueeze(2)                              # :341
    base_grid = torch.cat([arange, arange.transpose(1, 0)], dim=2)                      # :342  (x, y)
    base_grid = base_grid.unsqueeze(0).repeat(n, 1, 1, 1)                               # :343
    shift = shifts_xy.to(x.dtype).view(n, 1, 1, 2) * (2.0 / (h + 2 * pad))              # :345-350
    return F.grid_sample(xp, base_grid + shift, padding_mode="zeros", align_corners=False)   # :352-353


def random_shifts_grid_sample_traj(x, shifts_xy, pad):
    """data_utils.py:356-383: [n, t, c, h, w] flattened to n*t images, one shift per frame."""
    n, t = x.shape[:2]
    return random_shifts_grid_sample(x.reshape(n * t, *x.shape[2:]), shifts_xy, pad).view(n, t, *x.shape[2:])


def shift_crop(x, shifts_xy, pad):
    """out[i, c, y, x] = x[i, c, clamp(y + sy_i - pad, 0, h-1), clamp(x + sx_i - pad, 0, w-1)]."""
    n, c, h, w = x.shape
    ys = (torch.arange(h).view(1, h) + shifts_xy[:, 1].view(n, 1).long() - pad).clamp_(0, h - 1)      # [n, h]
    xs = (torch.arange(w).view(1, w) + shifts_xy[:, 0].view(n, 1).long() - pad).clamp_(0, w - 1)      # [n, w]
    idx = torch.arange(n).view(n, 1, 1)
    return x[idx, :, ys.view(n, h, 1), xs.view(n, 1, w)].permute(0, 3, 1, 2).contiguous()


def resize_nearest(x, hout, wout):
    """torchvision Resize(NEAREST) on a tensor = F.interpolate(mode='nearest') (data_utils.py:3598-3599): src index =
    min(floor(dst * in/out), in - 1) with the scale held in fp32 (ATen UpSample.h nearest_neighbor_compute_source_index)."""
    hin, win = x.shape[-2:]
    sh = torch.tensor(hin, dtype=torch.float32) / torch.tensor(hout, dtype=torch.float32)
    sw = torch.tensor(win, dtype=torch.float32) / torch.tensor(wout, dtype=torch.float32)
    ys = torch.floor(torch.arange(hout, dtype=torch.float32) * sh).long().clamp_(max=hin - 1)
    xs = torch.floor(torch.arange(wout, dtype=torch.float32) * sw).long().clamp_(max=win - 1)
    return x[..., ys.view(-1, 1), xs.view(1, -1)]
