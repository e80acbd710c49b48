"""Golden crops of CLIP's image transform (`image_processor`, openai CLIP `_transform(224)`), produced by torchvision + Pillow:

    python tests/golden/make_golden_image_fn.py  ->  tests/golden/image_fn.pt

openai CLIP is not a dependency here; its `_transform(n_px)` is Compose([Resize(n_px, BICUBIC), CenterCrop(n_px),
_convert_image_to_rgb, ToTensor(), Normalize(mean, std)]) in torchvision, restated below.  The file records the uint8 HWC crop
(Resize + CenterCrop: the only part that depends on Pillow) of every case; ToTensor + Normalize of a uint8 value is an
elementwise map that the tests rebuild with torch.  The inputs are not stored: `make_inputs()` regenerates them from a seeded
torch.Generator.  The crops are zlib-compressed to keep the file near 1 MB.
"""
from __future__ import annotations

import os
import zlib

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "image_fn.pt")

# (h, w): CALVIN static / gripper (200, 84), LIBERO (128), a downscale, the identity, both orientations of a non-square frame,
# a camera frame, a frame smaller than the kernel support, a large downscale
SHAPES = [(200, 200), (84, 84), (128, 128), (256, 256), (224, 224), (300, 173), (173, 300), (480, 640), (7, 5), (1000, 1000)]
KINDS = ("noise", "edges")
SEED = 20260101


def make_frame(h, w, kind, g):
    """uint8 [h, w, 3].  noise: uniform bytes on a band of rows and a band of columns (each a quarter of the frame, at a random
    place) over a flat background -- every output row and column sees noise, and the crop stays compressible.  edges:
    rectangles of 0 / 255 per channel (1 pixel up to half the frame on a side) on a random background level -- hard edges push
    the bicubic overshoot into both clamps of the 8-bit passes."""
    x = torch.randint(0, 256, (1, 1, 3), generator=g, dtype=torch.uint8).expand(h, w, 3).clone()
    if kind == "noise":
        bh, bw = max(2, h // 4), max(2, w // 4)
        y0, x0 = int(torch.randint(0, h - bh + 1, (1,), generator=g)), int(torch.randint(0, w - bw + 1, (1,), generator=g))
        x[y0:y0 + bh] = torch.randint(0, 256, (bh, w, 3), generator=g, dtype=torch.uint8)
        x[:, x0:x0 + bw] = torch.randint(0, 256, (h, bw, 3), generator=g, dtype=torch.uint8)
        return x
    for _ in range(24):
        y0, x0 = int(torch.randint(0, h, (1,), generator=g)), int(torch.randint(0, w, (1,), generator=g))
        dy, dx = int(torch.randint(1, max(2, h // 2), (1,), generator=g)), int(torch.randint(1, max(2, w // 2), (1,), generator=g))
        x[y0:y0 + dy, x0:x0 + dx] = torch.randint(0, 2, (3,), generator=g, dtype=torch.uint8) * 255
    return x


def make_inputs(seed=SEED, shapes=SHAPES):
    """[(name, uint8 [h, w, 3])] for every shape and kind, from one seeded generator."""
    g = torch.Generator().manual_seed(seed)
    return [(f"{h}x{w}_{kind}", make_frame(h, w, kind, g)) for h, w in shapes for kind in KINDS]


def clip_crop(frame):
    """Resize(224, BICUBIC) + CenterCrop(224) of CLIP's `_transform(224)` through Pillow: uint8 [h, w, 3] -> uint8 [224, 224, 3]."""
    from PIL import Image
    import torchvision.transforms as T
    tf = T.Compose([T.Resize(224, interpolation=T.InterpolationMode.BICUBIC), T.CenterCrop(224)])
    return torch.from_numpy(np.array(tf(Image.fromarray(frame.numpy())).convert("RGB")))


def main():
    import PIL
    import torchvision
    crops = {}
    for name, frame in make_inputs():
        c = clip_crop(frame)
        assert c.shape == (224, 224, 3) and c.dtype == torch.uint8
        crops[name] = torch.frombuffer(bytearray(zlib.compress(c.numpy().tobytes(), 9)), dtype=torch.uint8)
    torch.save({"seed": SEED, "shapes": SHAPES, "kinds": KINDS, "crops": crops,
                "versions": {"Pillow": PIL.__version__, "torchvision": torchvision.__version__, "torch": str(torch.__version__)}}, OUT)
    print(f"wrote {OUT}: {len(crops)} crops, {os.path.getsize(OUT)} bytes")


def load_crops(path=OUT):
    """{name: uint8 [224, 224, 3]} of the golden file, and the file's dict."""
    gold = torch.load(path)
    crops = {k: torch.frombuffer(bytearray(zlib.decompress(v.numpy().tobytes())), dtype=torch.uint8).view(224, 224, 3)
             for k, v in gold["crops"].items()}
    return crops, gold


if __name__ == "__main__":
    main()
