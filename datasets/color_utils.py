"""Image decoding of the disk loaders: the reference's ``read_image`` (datasets/color_utils.py:19-31).

The file is decoded to uint8 with PIL (the decoder behind ``imageio.imread`` for PNG and JPEG) and divided by 255 in
fp32.  An RGBA image is blended in fp32 in the reference's operation order: ``rgb * a + (1 - a)`` (onto white) when
``blend_a``, ``rgb * a`` (premultiplied, i.e. onto black) when not.  Then ``cv2.resize(img, img_wh)`` (bilinear) and
flatten to [H*W, 3].  With ``keep_alpha`` the resized alpha is appended as a fourth column, resized on its own so
that the three colour columns are exactly the reference's; ``--random_bg`` needs it to re-composite the target.

Grayscale, palette, 16-bit and other images the reference would mis-read raise ``ValueError``.
"""
from __future__ import annotations

import cv2
import numpy as np
from PIL import Image, ImageOps

_PNG_SIGNATURE = b'\x89PNG\r\n\x1a\n'


def decode_u8(img_path):
    """[H, W, 3|4] uint8 pixels of an 8-bit RGB or RGBA image."""
    with open(img_path, 'rb') as f:
        head = f.read(25)
    if head[:8] == _PNG_SIGNATURE and len(head) == 25 and head[24] != 8:
        raise ValueError(f"{img_path}: {head[24]}-bit PNG; the loaders read 8-bit RGB or RGBA images")
    with Image.open(img_path) as im:
        im = ImageOps.exif_transpose(im)
        if im.mode not in ('RGB', 'RGBA'):
            raise ValueError(f"{img_path}: image mode {im.mode!r}; the loaders read 8-bit RGB or RGBA images")
        return np.asarray(im, dtype=np.uint8)


def read_image(img_path, img_wh, blend_a=True, keep_alpha=False):
    img = decode_u8(img_path).astype(np.float32) / 255.0
    alpha = None
    if img.shape[2] == 4:
        alpha = img[..., -1:]
        img = img[..., :3] * alpha + (1 - alpha) if blend_a else img[..., :3] * alpha
    img = cv2.resize(img, img_wh).reshape(-1, 3)
    if keep_alpha and alpha is not None:
        a = cv2.resize(np.ascontiguousarray(alpha[..., 0]), img_wh).reshape(-1, 1)
        img = np.concatenate([img, a], 1)
    return img
