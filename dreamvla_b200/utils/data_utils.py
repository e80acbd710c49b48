"""Device-side pieces of the reference's collator (SURVEY.md 8f-2): CLIP's image transform, the random-shift augmentation and
the NEAREST depth resize that reference `utils/data_utils.py` runs on CPU data-loader workers (`image_fn` :175-179 / :1311-1312,
`RandomShiftsAug` :326-383, `depth_image_fn` :3588-3603, applied in `collator` :1337-1354).  Here they run on the GPU on the
already-transferred batch (`csrc/augment.cu`), so the loader can ship raw uint8 frames (`preprocess_image`) and un-augmented
tensors (`train.py --device_augment`).

Same class name, constructor and methods as the reference.  Randomness: the reference draws the integer shifts with
`torch.randint` from the worker's global CPU generator; here they come from `torch.randint` on the device (pass `generator=`
or explicit `shifts=` to control them) -- the distribution is the same (uniform on {0 | 1, ..., 2*pad}), the stream is not.
"""
from __future__ import annotations

import torch

from .. import _lib as L

# openai CLIP `_transform` Normalize constants
CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)
RAW_IMAGE_KEYS = ("images_primary", "images_wrist")

_luts = {}


def image_fn_lut(device):
    """fp32 [3, 256]: ToTensor + Normalize of every uint8 value, in torch's own arithmetic ((v / 255 - mean) / std), on `device`."""
    device = torch.device(device)
    lut = _luts.get(device)
    if lut is None:
        v = torch.arange(256, dtype=torch.float32) / 255
        mean, std = torch.tensor(CLIP_MEAN).view(3, 1), torch.tensor(CLIP_STD).view(3, 1)
        lut = _luts[device] = ((v - mean) / std).contiguous().to(device)
    return lut


def preprocess_image(frames, out_dtype=torch.float32, flip_vertical=False):
    """Reference `image_processor` (CLIP `_transform(224)`: Resize(224, BICUBIC), CenterCrop(224), ToTensor, Normalize) of
    uint8 RGB frames on the device, bit for bit what Pillow + torchvision give: uint8 [..., h, w, 3] -> [..., 3, 224, 224]
    `out_dtype` (fp32 / bf16).  `flip_vertical` flips every frame upside down first (LIBERO's agent view)."""
    if frames.dtype != torch.uint8 or frames.dim() < 3 or frames.shape[-1] != 3:
        raise ValueError(f"preprocess_image takes uint8 [..., h, w, 3] frames, got {frames.dtype} {tuple(frames.shape)}")
    lead, (h, w) = frames.shape[:-3], frames.shape[-3:-1]
    out = L.image_fn(frames.reshape(-1, h, w, 3).contiguous(), image_fn_lut(frames.device), out_dtype, flip_vertical)
    return out.view(*lead, 3, out.shape[-2], out.shape[-1])


class RandomShiftsAug:
    """Reference `RandomShiftsAug(pad)`: replicate-pad by `pad` and re-crop at a random integer offset per image."""

    def __init__(self, pad):
        self.pad = int(pad)

    def draw(self, n, device, low=0, generator=None):
        """int32 [n, 2] = (sx, sy), uniform on {low, ..., 2*pad} (reference :345-349 low = 0, :372-376 low = 1)."""
        return torch.randint(low, 2 * self.pad + 1, (n, 2), device=device, dtype=torch.int32, generator=generator)

    def forward(self, x, shifts=None, generator=None, out_dtype=None):
        """x [n, c, h, w] (reference :330-354); one shift per image."""
        n, c, h, w = x.shape
        assert h == w                                                                   # reference :332
        if shifts is None:
            shifts = self.draw(n, x.device, 0, generator)
        return L.shift_crop(x.contiguous(), shifts.to(device=x.device, dtype=torch.int32).contiguous(), self.pad, out_dtype)

    __call__ = forward

    def forward_traj(self, x, shifts=None, generator=None, out_dtype=None):
        """x [n, t, c, h, w] (reference :356-383); one shift per FRAME, drawn from {1, ..., 2*pad}."""
        n, t, c, h, w = x.shape
        assert h == w                                                                   # reference :359
        if shifts is None:
            shifts = self.draw(n * t, x.device, 1, generator)
        y = L.shift_crop(x.reshape(n * t, c, h, w).contiguous(), shifts.to(device=x.device, dtype=torch.int32).contiguous(),
                         self.pad, out_dtype)
        return y.view(n, t, c, h, w)


def depth_image_fn(depth, size=224, out_dtype=torch.float32):
    """Reference `depth_image_fn` (:3588-3603) for depth maps already on the device: float32 [..., H, W] -> [..., 1, size, size]
    by NEAREST resize (torchvision `Resize((224, 224), NEAREST)` on a tensor)."""
    d = depth.to(torch.float32).contiguous()
    return L.resize_nearest(d, size, size, out_dtype).unsqueeze(-3)


def augment_batch(batch, rgb_pad=-1, gripper_pad=-1, traj_cons=False, generator=None):
    """The augmentation block of the reference collator (:1337-1354) on a device batch dict (keys of
    `train_utils.batch_to_host_dict`).  With `traj_cons` the static / gripper RGB windows AND their depth windows go through
    `forward_traj` -- each call draws its own shifts, so an image and its depth map are shifted independently, exactly as the
    reference does; without it only the RGB windows are augmented, per image, through `forward`."""
    out = dict(batch)
    for pad, rgb_key, depth_key in ((rgb_pad, "images_primary", "depth_primary"), (gripper_pad, "images_wrist", "depth_wrist")):
        if pad is None or pad == -1 or rgb_key not in out:
            continue
        aug = RandomShiftsAug(pad)
        x = out[rgb_key]
        if traj_cons:
            out[rgb_key] = aug.forward_traj(x, generator=generator)
            if out.get(depth_key) is not None:
                out[depth_key] = aug.forward_traj(out[depth_key], generator=generator)
        else:
            bs, seq = x.shape[:2]
            out[rgb_key] = aug.forward(x.reshape(bs * seq, *x.shape[2:]), generator=generator).view(x.shape)
    return out


def prepare_batch(batch, rgb_pad=-1, gripper_pad=-1, traj_cons=False, device_augment=False, generator=None,
                  dtype=torch.bfloat16):
    """The image steps of the reference collator on a device batch, in its order: `image_fn` of every frame (:1311-1312), then
    the random shifts (:1337-1354).  RGB windows that arrive as uint8 [B, W, h, w, 3] (a loader that ships raw frames) are
    preprocessed to `dtype`; with `device_augment` the shifts follow (`augment_batch`).  Float windows pass unchanged.

    A raw-frame loader cannot have applied the shifts, so raw frames with a pad set but without `device_augment` raise."""
    raw = [k for k in RAW_IMAGE_KEYS if k in batch and batch[k].dtype == torch.uint8]
    pads = rgb_pad not in (None, -1) or gripper_pad not in (None, -1)
    if raw and pads and not device_augment:
        raise ValueError(f"the loader ships raw uint8 frames ({', '.join(raw)}) and rgb_pad / gripper_pad are set: the random "
                         "shifts can then only run on the device -- pass --device_augment")
    if raw:
        batch = dict(batch)
        for k in raw:
            batch[k] = preprocess_image(batch[k], dtype)
    if device_augment and pads:
        batch = augment_batch(batch, rgb_pad, gripper_pad, traj_cons, generator)
    return batch
