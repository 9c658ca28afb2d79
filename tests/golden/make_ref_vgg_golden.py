"""Record THE REFERENCE'S OWN VGGLoss (READ/criterions/vgg_loss.py) in tests/golden/ref_vgg_loss.npz: the loss and the input
gradient for net in ('caffe', 'pytorch') x optimized in (False, True), on seeded 2x3x48x64 images, so that
tests/test_vgg_loss_host.py can pin read_b200.vgg_loss.reference_loss (the restatement the GPU tests compare against) without the
reference.

Needs a checkout of the reference (READ) at READ_REFERENCE_ROOT (default /root/reference); CPU only, nothing is downloaded:

    python tests/golden/make_ref_vgg_golden.py

The weights are tests/vgg_util.seeded_features(): for 'caffe' they are written as the vgg_caffe_features.pth the reference loads
from a temporary save_dir; for 'pytorch' torchvision.models.vgg19 is replaced by a stand-in that returns them.  Both are
regenerated from the seed by the test, so only the results are committed.
"""
import copy
import os
import sys
import tempfile
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
OUT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.environ.get("READ_REFERENCE_ROOT", "/root/reference"))

from READ.criterions import vgg_loss as ref       # noqa: E402

import vgg_util                                   # noqa: E402

SHAPE = (2, 48, 64)
IMAGE_SEED = 5


def main():
    features = vgg_util.seeded_features()
    inp, tgt = vgg_util.seeded_images(*SHAPE, IMAGE_SEED)
    out = {}
    with tempfile.TemporaryDirectory() as save_dir:
        torch.save(copy.deepcopy(features), os.path.join(save_dir, "vgg_caffe_features.pth"))
        ref.torch.load = lambda path, **kw: torch.serialization.load(path, weights_only=False)
        ref.torchvision.models.vgg19 = lambda *a, **kw: types.SimpleNamespace(features=copy.deepcopy(features))
        for net in ("caffe", "pytorch"):
            for optimized in (False, True):
                crit = ref.VGGLoss(net=net, optimized=optimized, save_dir=save_dir)
                x = inp.clone().requires_grad_(True)
                loss = crit(x, tgt)
                loss.backward()
                tag = f"{net}_{'opt' if optimized else 'all'}"
                out[f"loss_{tag}"] = np.float64(loss.item())
                out[f"grad_{tag}"] = x.grad.numpy().astype(np.float32)
                print(tag, loss.item(), float(x.grad.abs().max()))
    np.savez_compressed(os.path.join(OUT, "ref_vgg_loss.npz"), **out)


if __name__ == "__main__":
    main()
