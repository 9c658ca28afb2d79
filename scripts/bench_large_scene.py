"""Cost of int32 index maps and of large clouds (scenes of more than 2^24 + 1 points get int32 maps, ops.index_map_dtype).  Three
measurements in one process, arms alternated over the rounds:
  (a) gather   the descriptor gather (NCHW f32) and sparse backward of the five C5 levels (8 crops of 256x256, 5M points) on float32
               maps and on int32 copies of the same ids; the bytes moved are the same, so equal within noise is expected;
  (b) step     the headless C5 step (tests/headless_util.py: MyRender -> ModelAndLoss -> vgg + 1e4 * huber -> Adam + SparseRMSprop,
               bf16_all with VGGLoss, eval mode) on a 5M-point scene (float maps) and on a 2^25-point one (int32 maps); only the
               rasterizer and the optimizer's scan of the touched flags grow with N;
  (c) frame    the fused 1920x1088 frame (NetAndTexture.render, bf16 engine) of a 2^25-point cloud.
   python scripts/bench_large_scene.py [--iters 20] [--rounds 5] [--out result.json]
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
from read_b200 import headless, ops, synth, train as rtrain, _lib as L    # noqa: E402
from read_b200.myrender import MyRender                                  # noqa: E402
from read_b200.texture import PointTexture                               # noqa: E402
from read_b200.unet import UNet                                          # noqa: E402
from read_b200.vgg_loss import VGGLoss                                   # noqa: E402
from bench_train_bf16 import card, ev, W, H, BC                          # noqa: E402
import headless_util as hu                                               # noqa: E402
import vgg_util                                                          # noqa: E402

N_SMALL, N_LARGE = 5_000_000, 2 ** 25
FW, FH = 1920, 1088


def timed(fn, iters):
    a, b = ev(), ev()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def summary(ms):
    return {k: {"rounds": v, "median": float(np.median(v)), "min": float(min(v)), "max": float(max(v))} for k, v in ms.items()}


def alternate(arms, rounds, iters):
    for fn in arms.values():                                     # warm-up of every shape
        timed(fn, 2)
    ms = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            ms[k].append(timed(fn, iters))
    return summary(ms)


def texture(n, dev):
    t = PointTexture(8, n)
    with torch.no_grad():
        t.texture_.copy_(torch.rand((1, 8, n), generator=torch.Generator().manual_seed(synth.SEED)))
    return t.to(dev)


def gather_arms(dev):
    scene = hu.scene(N_SMALL, W, H, depth=250.0)
    r = MyRender(device_outputs=True)
    r.update_ds([scene])
    maps, _ = r.render(hu.batch(W, H, list(range(BC))))
    ids_f = [v[:, 0].contiguous() for k, v in maps.items() if k != 'id']
    ids_i = [i.to(torch.int32) for i in ids_f]
    tex = torch.rand((N_SMALL, 8), device=dev)
    gos = [torch.randn((BC, 8) + tuple(i.shape[1:]), device=dev) for i in ids_f]
    acc, touched = torch.zeros((N_SMALL, 8), device=dev), torch.zeros(N_SMALL, dtype=torch.uint8, device=dev)

    def arm(ids):
        def fn():
            for i, go in zip(ids, gos):
                ops.gather_from_index(tex, i, L.FEAT_NCHW_F32)
                ops.gather_backward_sparse(go, i, N_SMALL, acc, touched)
        return fn
    return {"gather+sparse bwd, float32 maps": arm(ids_f), "gather+sparse bwd, int32 maps": arm(ids_i)}


def step_arm(n, sd, dev):
    scene = hu.scene(n, W, H, depth=250.0)
    r = MyRender()
    r.update_ds([scene])
    net = UNet()
    net.load_state_dict(sd, strict=True)
    net.train_precision = 'bf16_all'
    tex = texture(n, dev)
    model = headless.NetAndTexture(net, {0: tex})
    model.load_textures([0])
    model.to(dev).eval()
    loss_mod = hu.ModelAndLoss(model, VGGLoss(features=vgg_util.seeded_features()).to(dev))
    opt_net, opt_tex = torch.optim.Adam(net.parameters(), lr=1e-4), rtrain.SparseRMSprop([tex], lr=0.1)
    rng = np.random.default_rng(synth.SEED)
    data = hu.batch(W, H, rng.integers(0, 64, BC))
    target = torch.rand((BC, 3, H, W), generator=torch.Generator().manual_seed(7)).to(dev)

    def fn():
        loss = hu.forward_loss(r, loss_mod, data, target, None, dev, model.reg_loss)
        loss.backward()
        opt_net.step()
        opt_net.zero_grad()
        opt_tex.step()
    return fn, r.index_dtype


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

    out["gather"] = alternate(gather_arms(dev), args.rounds, args.iters)
    print(json.dumps({"gather": out["gather"]}), flush=True)

    sd = synth.synth_state_dict(synth.SEED)
    small, dt_small = step_arm(N_SMALL, sd, dev)
    large, dt_large = step_arm(N_LARGE, sd, dev)
    out["step"] = alternate({f"C5 step, {N_SMALL} points ({dt_small})": small, f"C5 step, {N_LARGE} points ({dt_large})": large},
                            args.rounds, max(args.iters // 4, 3))
    print(json.dumps({"step": out["step"]}), flush=True)
    del small, large
    torch.cuda.empty_cache()

    net = UNet()
    net.load_state_dict(sd, strict=True)
    model = headless.NetAndTexture(net, {0: texture(N_LARGE, dev)})
    model.load_textures([0])
    model.to(dev).eval()
    xyz = torch.from_numpy(synth.street_scene(N_LARGE, depth=250.0)).to(dev)
    proj, view = synth.camera_batch(FW, FH, [5])
    tm = torch.from_numpy(synth.total_matrix(proj, view)).to(dev)
    out["frame"] = alternate({f"fused {FW}x{FH} frame, {N_LARGE} points": lambda: model.render(xyz, tm, FW, FH, clone_output=False)},
                             args.rounds, args.iters)
    print(json.dumps({"frame": out["frame"]}), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
