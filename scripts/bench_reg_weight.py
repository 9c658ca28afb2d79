"""Cost of the descriptor regulariser (--reg_weight) on the sparse optimizer.  In one process, arms alternated over the rounds:
  (a) desc     the descriptor side alone at 5M and 2^25 points, with the touched set of a C5 step (index maps of 8 crops of 256x256,
               five levels, rendered from a synthetic scene): gather forward + backward of the five levels, reg_loss forward +
               backward and the optimizer step.  Ours: sparse gather backward, train._RegLoss and the dense-term step.  Torch: the
               dense gather backward, torch's expression with autograd's dense gradient and torch.optim.RMSprop.  Also the
               regulariser alone (reg_loss forward + backward + step, no gather), and the peak extra device memory of one iteration;
  (b) step     the headless C5 step (tests/headless_util.py: MyRender -> ModelAndLoss -> vgg + 1e4 * huber + reg_loss -> Adam + the
               descriptor optimizer, bf16_all with VGGLoss, eval mode, 5M points) at reg_weight 0 and 1e-3, with SparseRMSprop and
               with torch.optim.RMSprop (--dense_texture_optimizer).
A lower bound for the dense-term step: 7 x 32 B of HBM traffic per point at 3.35 TB/s (arithmetic, printed beside the times).
   python scripts/bench_reg_weight.py [--iters 20] [--rounds 5] [--out result.json]
Prints the card's name and power limit, then per arm the milliseconds of each round (CUDA events), median and range."""
import argparse
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tests"))
from read_b200 import headless, synth, train as rtrain, _lib as L      # noqa: E402
from read_b200.myrender import MyRender                                  # noqa: E402
from read_b200.texture import PointTexture                               # noqa: E402
from read_b200.unet import UNet                                          # noqa: E402
from read_b200.vgg_loss import VGGLoss                                   # noqa: E402
from bench_train_bf16 import card, W, H, BC                              # noqa: E402
from bench_large_scene import alternate                                  # noqa: E402
import headless_util as hu                                               # noqa: E402
import vgg_util                                                          # noqa: E402

N_SMALL, N_LARGE = 5_000_000, 2 ** 25
W_REG = 1e-3
HBM_BPS = 3.35e12


def texture(n, dev, reg_weight, sparse):
    t = PointTexture(8, n, reg_weight=reg_weight)
    with torch.no_grad():
        t.texture_.copy_(torch.rand((1, 8, n), generator=torch.Generator().manual_seed(synth.SEED)))
    t = t.to(dev)
    if sparse:
        rtrain.request_sparse_grad(t)
    return t


def level_maps(n, dev):
    """The five C5 levels' index maps of 8 crops of one synthetic scene of n points (the step's touched set)."""
    scene = hu.scene(n, W, H, depth=250.0)
    r = MyRender(device_outputs=True)
    r.update_ds([scene])
    maps, _ = r.render(hu.batch(W, H, list(range(BC))))
    ids = [v[:, :1].contiguous() for k, v in maps.items() if k != 'id']
    gos = [torch.randn((BC, 8) + tuple(i.shape[2:]), device=dev) for i in ids]
    return ids, gos


def desc_arms(n, dev):
    ids, gos = level_maps(n, dev)
    arms, mem = {}, {}
    for name, sparse in (("ours (sparse + dense-term step)", True), ("torch (dense grad + RMSprop)", False)):
        t = texture(n, dev, W_REG, sparse)
        opt = rtrain.SparseRMSprop(t, lr=0.1) if sparse else torch.optim.RMSprop(t.parameters(), lr=0.1)

        def full(t=t, opt=opt):
            loss = sum((t(i) * g).sum() for i, g in zip(ids, gos)) + t.reg_loss()
            loss.backward()
            opt.step()
            opt.zero_grad()

        def reg_only(t=t, opt=opt):
            t.reg_loss().backward()
            opt.step()
            opt.zero_grad()

        for fn in (full, full):                                  # optimizer state allocated before the memory reading
            fn()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        full()
        torch.cuda.synchronize()
        mem[name] = torch.cuda.max_memory_allocated() - base
        arms[f"{n} points, gather + reg_loss + step, {name}"] = full
        arms[f"{n} points, reg_loss + step only, {name}"] = reg_only
    return arms, mem


def step_arm(n, sd, dev, reg_weight, dense):
    scene = hu.scene(n, W, H, depth=250.0)
    r = MyRender()
    r.update_ds([scene])
    net = UNet()
    net.load_state_dict(sd, strict=True)
    net.train_precision = 'bf16_all'
    tex = texture(n, dev, reg_weight, not dense)
    model = headless.NetAndTexture(net, {0: tex})
    model.load_textures([0])
    model.to(dev).eval()
    loss_mod = hu.ModelAndLoss(model, VGGLoss(features=vgg_util.seeded_features()).to(dev))
    opt_net = torch.optim.Adam(net.parameters(), lr=1e-4)
    opt_tex = torch.optim.RMSprop(tex.parameters(), lr=0.1) if dense else rtrain.SparseRMSprop([tex], lr=0.1)
    rng = np.random.default_rng(synth.SEED)
    data = hu.batch(W, H, rng.integers(0, 64, BC))
    target = torch.rand((BC, 3, H, W), generator=torch.Generator().manual_seed(7)).to(dev)

    def fn():
        loss = hu.forward_loss(r, loss_mod, data, target, None, dev, model.reg_loss)
        loss.backward()
        opt_net.step()
        opt_net.zero_grad()
        opt_tex.step()
        opt_tex.zero_grad()
    return fn


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    L.require_device(0)
    out = {"card": card()}
    print(json.dumps(out["card"]), flush=True)

    for n in (N_SMALL, N_LARGE):
        arms, mem = desc_arms(n, dev)
        res = alternate(arms, args.rounds, args.iters)
        bound_ms = 7 * 32 * n / HBM_BPS * 1e3
        out[f"desc_{n}"] = {"times": res, "peak_extra_bytes": mem, "dense_step_lower_bound_ms": bound_ms}
        print(json.dumps({f"desc_{n}": out[f"desc_{n}"]}), flush=True)
        del arms
        torch.cuda.empty_cache()

    sd = synth.synth_state_dict(synth.SEED)
    steps = {}
    for w in (0.0, W_REG):
        for dense in (False, True):
            steps[f"C5 step, {N_SMALL} points, reg_weight {w}, {'torch RMSprop' if dense else 'SparseRMSprop'}"] = \
                step_arm(N_SMALL, sd, dev, w, dense)
    out["step"] = alternate(steps, args.rounds, max(args.iters // 4, 3))
    print(json.dumps({"step": out["step"]}), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
