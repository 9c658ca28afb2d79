"""Seeded image pairs for the masked (partialconv=True) VGG loss tests: the three target kinds the golden fixture records."""
import torch

import vgg_util

KINDS = ("holes", "dense", "zero")


def masked_pair(kind, B, H, W, seed):
    """(input, target) [B, 3, H, W] f32 in [0, 1).  'holes': the target has zeroed rectangles (one inside the image, one on the
    border, per image), so its validity mask has holes; 'dense': no zero pixel, only the border windows are rescaled; 'zero': an
    all-zero target, whose mask is empty."""
    x, t = vgg_util.seeded_images(B, H, W, seed)
    t = 0.01 + 0.98 * t                                   # no pixel sums to 0 by chance
    if kind == "holes":
        for b in range(B):
            y0, x0 = (H // 4 + 3 * b) % H, (W // 3 + 5 * b) % W
            t[b, :, y0:y0 + H // 3, x0:x0 + W // 4] = 0
            if b % 2:
                t[b, :, H - H // 5:, :W // 3] = 0
            else:
                t[b, :, :H // 6, W - W // 5:] = 0
    elif kind == "zero":
        t.zero_()
    elif kind != "dense":
        raise ValueError(kind)
    return x, t
