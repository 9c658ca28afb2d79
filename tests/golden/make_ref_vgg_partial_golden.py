"""Record THE REFERENCE'S OWN masked VGG loss (READ/criterions/vgg_loss.py: VGGLoss(partialconv=True) and VGGLossMix) in
tests/golden/ref_vgg_loss_partial.npz, so that tests/test_vgg_partial_host.py can pin read_b200.vgg_loss.reference_loss's partial
path (the restatement the GPU tests compare against) without the reference:

* VGGLoss(partialconv=True): the loss and the input gradient for net in ('caffe', 'pytorch') x optimized in (False, True) x the
  target kinds of tests/vgg_partial_util.py (zeroed rectangles, no zeros, all zeros), on seeded 2x3x36x52 images;
* VGGLossMix(weight=0.3): the loss and the input gradient on the 'holes' pair;
* the state_dict keys of both classes.

Needs a checkout of the reference (READ) at READ_REFERENCE_ROOT (default /root/reference); CPU only, nothing is downloaded:

    python tests/golden/make_ref_vgg_partial_golden.py

The weights are tests/vgg_util.seeded_features(), handed to the reference as make_ref_vgg_golden.py does.  VGGLossMix builds its
losses with the default save_dir, a relative path, so the file is also written there under a temporary working directory.
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

import vgg_partial_util                           # noqa: E402
import vgg_util                                   # noqa: E402

SHAPE = (2, 36, 52)
IMAGE_SEED = 12
MIX_WEIGHT = 0.3


def _record(out, tag, crit, inp, tgt):
    x = inp.clone().requires_grad_(True)
    loss = crit(x, tgt)
    loss.backward()
    out[f"loss_{tag}"] = np.float64(loss.item())
    out[f"grad_{tag}"] = x.grad.numpy().astype(np.float32)
    print(tag, loss.item(), float(x.grad.abs().max()))


def main():
    features = vgg_util.seeded_features()
    out = {}
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as work:
        save_dir = os.path.join(work, ".cache", "torch", "models")
        os.makedirs(save_dir)
        torch.save(copy.deepcopy(features), os.path.join(save_dir, "vgg_caffe_features.pth"))
        ref.torch.load = lambda path, **kw: torch.serialization.load(path, weights_only=False)
        ref.torchvision.models.vgg19 = lambda *a, **kw: types.SimpleNamespace(features=copy.deepcopy(features))
        for kind in vgg_partial_util.KINDS:
            inp, tgt = vgg_partial_util.masked_pair(kind, *SHAPE, IMAGE_SEED)
            for net in ("caffe", "pytorch"):
                for optimized in (False, True):
                    crit = ref.VGGLoss(net=net, partialconv=True, optimized=optimized, save_dir=save_dir)
                    _record(out, f"{kind}_{net}_{'opt' if optimized else 'all'}", crit, inp, tgt)
        out["keys_partial"] = np.array(sorted(crit.state_dict()))
        os.chdir(work)
        try:
            mix = ref.VGGLossMix(weight=MIX_WEIGHT)
        finally:
            os.chdir(cwd)
        inp, tgt = vgg_partial_util.masked_pair("holes", *SHAPE, IMAGE_SEED)
        _record(out, "mix", mix, inp, tgt)
        out["keys_mix"] = np.array(sorted(mix.state_dict()))
    np.savez_compressed(os.path.join(OUT, "ref_vgg_loss_partial.npz"), **out)


if __name__ == "__main__":
    main()
