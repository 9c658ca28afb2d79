"""The cost of torch.use_deterministic_algorithms(True) on the C5 training step (8 crops of 256x256, 5M points, bf16_all, per-item
train-mode BatchNorm, VGGLoss on our kernels, Adam on the net, sparse RMSprop on the descriptors), with the flag off and on
alternated over the rounds in one process, and each reduction's default kernel against its deterministic variant at the C5 shapes.
   python scripts/bench_train_deterministic.py [--steps 10] [--rounds 3] [--out result.json]
Prints the card's name and power limit, the step time per round in each arm, and per kernel shape the default and deterministic
times (CUDA events over 20 calls after a warm-up)."""
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
from read_b200 import synth, ops, blocks, vgg_loss, _lib as L     # noqa: E402
from bench_train_bf16 import make_model, card, ev, N, W, H, BC, LEVELS   # noqa: E402
import vgg_util                                                     # noqa: E402


def timeit(fn, reps=20):
    fn()
    torch.cuda.synchronize()
    a, b = ev(), ev()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def kernels(dev):
    """Default vs deterministic time (ms) of each reduction at its C5 shapes."""
    lib, st = L.load(), L.stream_ptr()
    g = torch.Generator().manual_seed(0)
    res = {}
    for l in range(LEVELS):                                         # gather backward, dense and sparse, per pyramid level
        h, w = H >> l, W >> l
        ids = torch.randint(0, N, (BC, h, w), generator=g).float()
        ids[torch.rand((BC, h, w), generator=g) < 0.5] = 0          # empty pixels carry id 0
        ids, go = ids.to(dev), torch.randn((BC, 8, h, w), generator=g).to(dev)
        acc, touched = torch.zeros((N, 8), device=dev), torch.zeros(N, dtype=torch.uint8, device=dev)
        ws = ops.det_workspace(lib.read_gather_backward_det_workspace_bytes(BC, 8, h, w, N), dev, "bench")
        res[f"gather_bwd_dense L{l} {BC}x{h}x{w}"] = [
            timeit(lambda: L.check(lib.read_gather_backward(go.data_ptr(), ids.data_ptr(), BC, 8, h, w, N, acc.data_ptr(), st))),
            timeit(lambda: L.check(lib.read_gather_backward_det(go.data_ptr(), ids.data_ptr(), BC, 8, h, w, N, acc.data_ptr(),
                                                                ws.data_ptr(), st)))]
        res[f"gather_bwd_sparse L{l} {BC}x{h}x{w}"] = [
            timeit(lambda: L.check(lib.read_gather_backward_sparse(go.data_ptr(), ids.data_ptr(), BC, 8, h, w, N, acc.data_ptr(),
                                                                   touched.data_ptr(), st))),
            timeit(lambda: L.check(lib.read_gather_backward_sparse_det(go.data_ptr(), ids.data_ptr(), BC, 8, h, w, N, acc.data_ptr(),
                                                                       touched.data_ptr(), ws.data_ptr(), st)))]
    for C, s in ((32, 256), (64, 128), (128, 64), (256, 32)):         # the stacks' gate passes, per item (8 items)
        P = s * s
        dy = torch.randn((BC * P, C), generator=g).bfloat16().to(dev)
        fm = torch.randn((BC * P, 2 * C), generator=g).bfloat16().to(dev)
        dfm = torch.empty_like(fm)
        v = torch.rand((8, BC, C), generator=g).to(dev) + 0.5
        red = torch.zeros((4, BC, C), device=dev)
        ws = ops.det_workspace(lib.read_gate_det_workspace_bytes(BC, C), dev, "bench")
        p = lambda t: t.data_ptr()
        args = lambda: (p(dy), p(fm), BC, P, C, 1, p(v[0, 0]), p(v[1, 0]), p(v[2]), p(v[3]), p(v[4]))
        res[f"gate_bwd_items C={C} {BC}x{s}x{s}"] = [
            timeit(lambda: L.check(lib.read_gate_backward_batch_stats_items(*args(), p(v[5]), p(v[6]), p(dfm), p(red[0, 0]),
                                                                            p(red[1, 0]), st))),
            timeit(lambda: L.check(lib.read_gate_backward_batch_stats_items_det(*args(), p(v[5]), p(v[6]), p(dfm), p(red[0, 0]),
                                                                                p(red[1, 0]), p(ws), st)))]
        rargs = lambda: (p(dy), p(fm), BC, P, C, 1, p(v[0, 0]), p(v[1, 0]), p(v[3]), p(v[4]), p(red[2]), p(red[3]))
        res[f"bn_bwd_reduce_items C={C} {BC}x{s}x{s}"] = [
            timeit(lambda: L.check(lib.read_bn_backward_reduce_items(*rargs(), st))),
            timeit(lambda: L.check(lib.read_bn_backward_reduce_items_det(*rargs(), p(ws), st)))]
    for cin, C, k, stride, s in ((32, 32, 3, 1, 256), (64, 64, 3, 1, 128), (128, 128, 3, 1, 64), (8, 32, 3, 1, 256),
                                 (64, 32, 1, 1, 256), (32, 64, 3, 2, 128), (64, 32, 4, 2, 256)):
        Hi, Ho = s, s // stride                                     # s: the input size
        dfm = torch.randn((BC, Ho, Ho, 2 * C), generator=g).bfloat16().to(dev)
        x = torch.randn((BC, Hi, Hi, cin), generator=g).bfloat16().to(dev)
        dw = torch.zeros((2, C, cin, k, k), device=dev)
        ws = ops.det_workspace(lib.read_conv_wgrad_det_workspace_bytes(BC, Ho, Ho, C, cin, k, stride), dev, "bench")
        res[f"wgrad {k}x{k}/s{stride} {cin}->{C} out {BC}x{Ho}x{Ho}"] = [
            timeit(lambda: L.check(lib.read_conv_wgrad(dfm.data_ptr(), x.data_ptr(), BC, Hi, Hi, Ho, Ho, C, cin, k, stride,
                                                       dw[0].data_ptr(), dw[1].data_ptr(), st))),
            timeit(lambda: L.check(lib.read_conv_wgrad_det(dfm.data_ptr(), x.data_ptr(), BC, Hi, Hi, Ho, Ho, C, cin, k, stride,
                                                           dw[0].data_ptr(), dw[1].data_ptr(), ws.data_ptr(), st)))]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    L.require_device(0)
    torch.backends.cudnn.benchmark = False
    os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    xyz = torch.from_numpy(synth.street_scene(N)).to(dev)
    store = ops.SortedPoints(xyz)
    pyr = ops.Pyramid(BC, W, H, LEVELS, dev)
    rng = np.random.default_rng(synth.SEED)
    mats = torch.stack([torch.from_numpy(synth.total_matrix(*synth.crop_cameras(W, H, rng.integers(0, 64, BC), rng)))
                        for _ in range(3 + args.steps)]).to(dev)
    target = torch.rand((BC, 3, H, W), generator=torch.Generator().manual_seed(7)).to(dev)
    keys = ["uv_1d_p1"] + [f"uv_1d_p1_ds{l}" for l in range(1, LEVELS)]
    crit = vgg_loss.VGGLoss(features=vgg_util.seeded_features()).to(dev)
    sd = synth.synth_state_dict(synth.SEED)
    runs = {arm: make_model(sd, "bf16_all", dev, True, True) for arm in ("off", "on")}

    def step(r, m):
        pyr.clear()
        ops.raster_project_sorted(pyr, store, m)
        ops.raster_derive(pyr)
        inputs = {k: ops.zbuf_resolve(pyr, l, want_depth=False)[0].unsqueeze(1) for l, k in enumerate(keys)}
        inputs["id"] = torch.zeros(BC, dtype=torch.long)
        loss = crit(r["model"](inputs), target)
        loss.backward()
        r["opt_net"].step()
        r["opt_tex"].step()
        r["opt_net"].zero_grad(set_to_none=True)
        return loss

    for arm, r in runs.items():
        torch.use_deterministic_algorithms(arm == "on")
        for s in range(3):
            step(r, mats[s])
    torch.cuda.synchronize()
    ms = {arm: [] for arm in runs}
    for _ in range(args.rounds):
        for arm, r in runs.items():
            torch.use_deterministic_algorithms(arm == "on")
            torch.cuda.synchronize()
            a, b = ev(), ev()
            a.record()
            for s in range(args.steps):
                step(r, mats[3 + s])
            b.record()
            torch.cuda.synchronize()
            ms[arm].append(a.elapsed_time(b) / args.steps)
    torch.use_deterministic_algorithms(False)
    kern = kernels(dev)
    out = {"card": card(), "step_ms": ms, "step_ms_median": {k: float(np.median(v)) for k, v in ms.items()},
           "kernels_ms_default_det": kern}
    print(json.dumps(out["card"]))
    for arm in ms:
        print(f"C5 step, flag {arm}: " + ", ".join(f"{t:.2f}" for t in ms[arm]) + f" ms (median {out['step_ms_median'][arm]:.2f})")
    for name, (a, b) in kern.items():
        print(f"  {name:48s} default {a * 1e3:8.1f} us   deterministic {b * 1e3:8.1f} us")
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
