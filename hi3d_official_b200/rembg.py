"""The two rembg calls of the reference's stage 1 (pipeline_i2v_eval_v01.py:153-168), `rembg.remove(image,
session=rembg.new_session())`, with the U^2-Net of u2net.py in place of onnxruntime and rembg's u2net.onnx.

This restates rembg 2.0.57's `bg.remove` and `U2netSession.predict` for that call only (no alpha matting, mask-only output,
background colour or other models: nothing here uses them).  Every step except the network is the same PIL / numpy call in the
same order: EXIF orientation, RGB -> 320 x 320 LANCZOS -> / max -> ImageNet mean / std in float64 -> float32, the network's
sigmoid(d0), min-max normalisation in float32, a truncating uint8 cast, LANCZOS back to the image size, and rembg's
`naive_cutout` (the image composited over transparent black through the mask).
"""
from __future__ import annotations

import os
from typing import Callable, Dict, Optional

import numpy as np
import torch

DEFAULT_WEIGHTS = os.path.join("ckpts", "u2net.pth")
SIZE = (320, 320)
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


class U2netSession:
    """`net`: the network, a callable from a float32 (1, 3, 320, 320) tensor to (1, 320, 320) probabilities."""

    def __init__(self, net: Callable[[torch.Tensor], torch.Tensor]):
        self.net = net

    def normalize(self, img) -> np.ndarray:
        from PIL import Image
        im = img.convert("RGB").resize(SIZE, Image.LANCZOS)
        im_ary = np.array(im)
        im_ary = im_ary / np.max(im_ary)
        tmp = np.zeros((im_ary.shape[0], im_ary.shape[1], 3))
        for c in range(3):
            tmp[:, :, c] = (im_ary[:, :, c] - MEAN[c]) / STD[c]
        return np.expand_dims(tmp.transpose((2, 0, 1)), 0).astype(np.float32)

    def predict(self, img):
        """The (img.size) "L" mask of U2netSession.predict."""
        from PIL import Image
        x = torch.from_numpy(self.normalize(img))
        pred = self.net(x)
        pred = pred.detach().float().cpu().numpy() if isinstance(pred, torch.Tensor) else np.asarray(pred, dtype=np.float32)
        pred = pred.reshape(SIZE[1], SIZE[0])
        ma, mi = np.max(pred), np.min(pred)
        pred = (pred - mi) / (ma - mi)
        mask = Image.fromarray((pred * 255).astype("uint8"), mode="L")
        return mask.resize(img.size, Image.LANCZOS)


def new_session(state_dict: Optional[Dict[str, torch.Tensor]] = None, device="cuda") -> U2netSession:
    """rembg.new_session() for its default model: U^2-Net on this package's kernels, from `state_dict` or from
    ckpts/u2net.pth under the working directory (U-2-Net's released weights).  Raises FileNotFoundError without either."""
    from .u2net import U2NetTower, load_u2net
    if state_dict is None:
        if not os.path.exists(DEFAULT_WEIGHTS):
            raise FileNotFoundError(f"{DEFAULT_WEIGHTS} not found: U^2-Net weights are needed for background removal")
        state_dict = load_u2net(DEFAULT_WEIGHTS)
    return U2netSession(U2NetTower(state_dict, device=device))


def remove(img, session: U2netSession):
    """rembg.remove(img, session=session) for a PIL image: the RGBA cut-out at img's (EXIF-corrected) size."""
    from PIL import Image, ImageOps
    img = ImageOps.exif_transpose(img)                    # fix_image_orientation
    mask = session.predict(img)
    empty = Image.new("RGBA", img.size, 0)                # naive_cutout
    return Image.composite(img, empty, mask)
