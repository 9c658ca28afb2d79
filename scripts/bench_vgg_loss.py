"""C5 training step (8 crops of 256x256, 5M points, the net in train() under 'bf16_all' with per-item BatchNorm: one batched net
call per step) with three losses, alternating in one process so that clock drift hits all alike: F.l1_loss (bench.py's loss), the
reference's VGG loss in torch (fp32, cuDNN defaults: TF32 convolutions) and read_b200.vgg_loss.VGGLoss (bf16 on our kernels).
Both VGG arms use the same seeded weights (the pretrained ones cannot be downloaded; the cost does not depend on their values).
    python scripts/bench_vgg_loss.py [--steps 10] [--rounds 3] [--out result.json]
Prints the card's name and power limit, per arm the step medians and their spread over rounds, the loss's forward + backward alone
on the 8 output crops, per conv of the loss its forward (2 x 8 images) and input-gradient (8 images) time and TFLOP/s (FLOPs from
shapes, real channels), and the time of each new kernel with its share of 3.35 TB/s (bytes from shapes).

--partialconv measures the masked loss (partialconv=True) instead: the target has zeroed holes and both images are multiplied by
their mask as ModelAndLoss(use_mask=True) does, and the arms are VGGLoss(partialconv=True) and VGGLoss() on our kernels and the
torch masked loss; then the loss's forward + backward alone per arm, and the partial kernels against their plain counterparts at
conv1_1's shapes."""
import argparse
import json
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tests"))
from read_b200 import synth, ops, blocks, vgg_loss, _lib as L     # noqa: E402
from bench_train_bf16 import make_model, card, ev, N, W, H, BC, LEVELS   # noqa: E402
import vgg_util                                                     # noqa: E402

HBM = 3.35e12


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = ev(), ev()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    ap.add_argument("--partialconv", action="store_true")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    L.require_device(0)
    xyz = torch.from_numpy(synth.street_scene(N)).to(dev)
    store = ops.SortedPoints(xyz)
    pyr = ops.Pyramid(BC, W, H, LEVELS, dev)
    rng = np.random.default_rng(synth.SEED)
    mats = torch.stack([torch.from_numpy(synth.total_matrix(*synth.crop_cameras(W, H, rng.integers(0, 64, BC), rng)))
                        for _ in range(3 + args.steps)]).to(dev)
    target = torch.rand((BC, 3, H, W), generator=torch.Generator().manual_seed(7)).to(dev)
    mask = None
    if args.partialconv:                             # a hole per crop, at a different place in each
        mask = torch.ones((BC, 1, H, W), device=dev)
        for b in range(BC):
            y0, x0 = 16 * b, 24 * b
            mask[b, :, y0:y0 + H // 3, x0:x0 + W // 4] = 0
        target = target * mask
    keys = ["uv_1d_p1"] + [f"uv_1d_p1_ds{l}" for l in range(1, LEVELS)]
    ids0 = torch.zeros(BC, dtype=torch.long)
    sd = synth.synth_state_dict(synth.SEED)
    crit = vgg_loss.VGGLoss(features=vgg_util.seeded_features()).to(dev)
    torch_vgg = lambda out, t: vgg_loss.reference_loss(crit.vgg19, crit.mean_, crit.std_, crit.layers, out, t)
    losses = {"l1": F.l1_loss, "vgg_torch": torch_vgg, "vgg_ours": crit}
    if args.partialconv:
        crit_p = vgg_loss.VGGLoss(partialconv=True, features=vgg_loss.partial_features(vgg_util.seeded_features())).to(dev)
        torch_p = lambda out, t: vgg_loss.reference_loss(crit_p.vgg19, crit_p.mean_, crit_p.std_, crit_p.layers, out, t)
        losses = {"vgg_ours": crit, "vgg_ours_partial": crit_p, "vgg_torch_partial": torch_p}
    runs = {k: make_model(sd, "bf16_all", dev, True, True) for k in losses}

    def step(r, lossf, m):
        pyr.clear()
        ops.raster_project_sorted(pyr, store, m)
        ops.raster_derive(pyr)
        inputs = {k: ops.zbuf_resolve(pyr, l, want_depth=False)[0].unsqueeze(1) for l, k in enumerate(keys)}
        inputs["id"] = ids0
        out = r["model"](inputs)
        loss = lossf(out if mask is None else out * mask, target)
        loss.backward()
        r["opt_net"].step()
        r["opt_tex"].step()
        r["opt_net"].zero_grad(set_to_none=True)

    for k, r in runs.items():
        for s in range(3):
            step(r, losses[k], mats[s])
    torch.cuda.synchronize()
    ms = {k: [] for k in runs}
    for _ in range(args.rounds):
        for k, r in runs.items():
            torch.cuda.synchronize()
            a, b = ev(), ev()
            a.record()
            for s in range(args.steps):
                step(r, losses[k], mats[3 + s])
            b.record()
            torch.cuda.synchronize()
            ms[k].append(a.elapsed_time(b) / args.steps)

    # the loss alone: forward + backward to the 8 output crops
    out = torch.rand((BC, 3, H, W), generator=torch.Generator().manual_seed(8)).to(dev)
    if mask is not None:
        out = out * mask
    alone = {}
    for k in [k for k in losses if k != "l1"]:
        def fb(k=k):
            x = out.clone().requires_grad_(True)
            losses[k](x, target).backward()
        alone[k] = [timed(fb, args.reps) for _ in range(args.rounds)]

    def summary(v):
        return {"median": round(float(np.median(v)), 2), "min": round(min(v), 2), "max": round(max(v), 2)}

    if args.partialconv:
        res = {"card": card(), "workload": "C5 step, 8 x 256^2 crops with holes, output and target masked, bf16_all, per-item "
               "BatchNorm, one net call per step", "steps": args.steps, "rounds": args.rounds,
               "step_ms": {k: summary(v) for k, v in ms.items()},
               "loss_fwd_bwd_ms": {k: summary(v) for k, v in alone.items()},
               "kernels": partial_kernels(crit_p, out, target, dev, args.reps)}
        print(json.dumps(res, indent=1))
        if args.out:
            with open(args.out, "w") as f:
                json.dump(res, f, indent=1)
        return

    # per conv and per new kernel at the C5 shapes
    lib, st = L.load(), L.stream_ptr()
    steps = crit.steps()
    pk = crit.filters(dev)
    zeros = torch.zeros(256, device=dev)
    ws = torch.empty(lib.read_vgg_workspace_bytes(), dtype=torch.uint8, device=dev)
    term = torch.zeros(1, dtype=torch.float64, device=dev)
    g1 = torch.ones(1, device=dev)
    layers = []
    for i, (s, (h, w)) in enumerate(zip(steps, vgg_loss.layer_sizes(steps, H, W))):
        cin = 8 if s.cin == 3 else s.cin
        x = torch.randn((2 * BC, h, w, cin), device=dev).to(torch.bfloat16)
        raw = torch.empty((2 * BC, h, w, s.cout), dtype=torch.bfloat16, device=dev)
        fwd = timed(lambda: blocks._launch(lib, x, s.cout // 2, pk[i]['w_tc'], (zeros,) * 4, False, L.OUT_RAW_NHWC, raw), args.reps)
        dy = torch.randn((BC, h, w, s.cout), device=dev).to(torch.bfloat16)
        dx = torch.empty((BC, h, w, cin), dtype=torch.bfloat16, device=dev)
        if i == 0:
            bwd = timed(lambda: L.check(lib.read_conv3x3_dgrad_cin8(dy.data_ptr(), pk[0]['wf'].data_ptr(), pk[0]['wm'].data_ptr(), BC,
                                                                     h, w, s.cout // 2, dx.data_ptr(), st)), args.reps)
        else:
            bwd = timed(lambda: blocks._launch(lib, dy, s.cin // 2, pk[i]['w_dgrad'], (zeros,) * 4, False, L.OUT_RAW_NHWC, dx),
                        args.reps)
        nxt = torch.empty((2 * BC, h // 2, w // 2, s.cout) if s.pool else (2 * BC, h, w, s.cout), dtype=torch.bfloat16, device=dev)
        code = torch.empty((BC, h, w, s.cout), dtype=torch.int8, device=dev)
        post = timed(lambda: L.check(lib.read_vgg_post(raw.data_ptr(), BC, h, w, s.cout, pk[i]['bias'].data_ptr(), int(s.pool),
                                                       nxt.data_ptr(), code.data_ptr(), term.data_ptr(), 1e-9, ws.data_ptr(), st)),
                     args.reps)
        up = torch.randn((BC, h // 2, w // 2, s.cout) if s.pool else (BC, h, w, s.cout), device=dev).to(torch.bfloat16)
        din = timed(lambda: L.check(lib.read_vgg_dgrad_in(up.data_ptr(), int(s.pool), code.data_ptr(), BC, h, w, s.cout,
                                                          g1.data_ptr(), 1e-9, dy.data_ptr(), st)), args.reps)
        e = BC * h * w * s.cout
        post_bytes = 2 * e * 2 + nxt.numel() * 2 + e
        din_bytes = e + up.numel() * 2 + e * 2
        flops_f = 2.0 * 2 * BC * h * w * s.cin * s.cout * 9
        flops_b = 2.0 * BC * h * w * s.cin * s.cout * 9
        layers.append({"conv": s.conv, "hw": [h, w], "cin": s.cin, "cout": s.cout, "fwd_ms": round(fwd, 4),
                       "fwd_tflops": round(flops_f / fwd / 1e9, 1), "dgrad_ms": round(bwd, 4),
                       "dgrad_tflops": round(flops_b / bwd / 1e9, 1), "post_ms": round(post, 4),
                       "post_hbm_share": round(post_bytes / HBM / (post * 1e-3), 3), "dgrad_in_ms": round(din, 4),
                       "dgrad_in_hbm_share": round(din_bytes / HBM / (din * 1e-3), 3)})
    img = torch.rand((BC, 3, H, W), device=dev)
    x8 = torch.empty((2 * BC, H, W, 8), dtype=torch.bfloat16, device=dev)
    mean, std = crit.mean_.contiguous(), crit.std_.contiguous()
    norm = timed(lambda: L.check(lib.read_vgg_normalize(img.data_ptr(), target.data_ptr(), BC, H, W, mean.data_ptr(), std.data_ptr(),
                                                        x8.data_ptr(), st)), args.reps)
    grad = torch.empty((BC, 3, H, W), device=dev)
    igrad = timed(lambda: L.check(lib.read_vgg_image_grad(x8.data_ptr(), BC, H, W, std.data_ptr(), grad.data_ptr(), st)), args.reps)
    kernels = {"vgg_normalize": {"ms": round(norm, 4), "hbm_share": round((2 * BC * H * W * (12 + 16)) / HBM / (norm * 1e-3), 3)},
               "vgg_image_grad": {"ms": round(igrad, 4), "hbm_share": round((BC * H * W * (16 + 12)) / HBM / (igrad * 1e-3), 3)}}

    res = {"card": card(), "workload": "C5 step, 8 x 256^2 crops, bf16_all, per-item BatchNorm, one net call per step",
           "steps": args.steps, "rounds": args.rounds,
           "step_ms": {k: {"median": round(float(np.median(v)), 2), "min": round(min(v), 2), "max": round(max(v), 2)}
                       for k, v in ms.items()},
           "loss_fwd_bwd_ms": {k: {"median": round(float(np.median(v)), 2), "min": round(min(v), 2), "max": round(max(v), 2)}
                               for k, v in alone.items()},
           "conv_layers": layers, "kernels": kernels}
    print(json.dumps(res, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


def partial_kernels(crit, out, target, dev, reps):
    """The partial kernels and their plain counterparts at conv1_1's C5 shapes (8 pairs of 256^2, 64 channels): time, bytes they
    must move and their share of 3.35 TB/s.  Alternated in one loop so that clock drift hits both alike."""
    lib, st = L.load(), L.stream_ptr()
    n, C = BC, 64
    mean, std = crit.mean_.contiguous(), crit.std_.contiguous()
    bias = crit.filters(dev)[0]['bias']
    x8 = torch.empty((2 * n, H, W, 8), dtype=torch.bfloat16, device=dev)
    m8 = torch.empty((n, H, W), dtype=torch.uint8, device=dev)
    L.check(lib.read_vgg_normalize_masked(out.data_ptr(), target.data_ptr(), n, H, W, mean.data_ptr(), std.data_ptr(), x8.data_ptr(),
                                          m8.data_ptr(), st))
    raw = torch.randn((2 * n, H, W, C), device=dev).to(torch.bfloat16)
    nxt = torch.empty_like(raw)
    code = torch.empty((n, H, W, C), dtype=torch.int8, device=dev)
    ws = torch.empty(lib.read_vgg_workspace_bytes(), dtype=torch.uint8, device=dev)
    term = torch.zeros(1, dtype=torch.float64, device=dev)
    g1 = torch.ones(1, device=dev)
    up = torch.randn((n, H, W, C), device=dev).to(torch.bfloat16)
    dy = torch.empty_like(up)
    grad = torch.empty((n, 3, H, W), device=dev)
    p, e = n * H * W, n * H * W * C
    arms = {
        "vgg_normalize": (lambda: L.check(lib.read_vgg_normalize(out.data_ptr(), target.data_ptr(), n, H, W, mean.data_ptr(),
                                                                 std.data_ptr(), x8.data_ptr(), st)), 2 * p * (12 + 16)),
        "vgg_normalize_masked": (lambda: L.check(lib.read_vgg_normalize_masked(out.data_ptr(), target.data_ptr(), n, H, W,
                                                                               mean.data_ptr(), std.data_ptr(), x8.data_ptr(),
                                                                               m8.data_ptr(), st)), 2 * p * (12 + 16) + p),
        "vgg_post": (lambda: L.check(lib.read_vgg_post(raw.data_ptr(), n, H, W, C, bias.data_ptr(), 0, nxt.data_ptr(),
                                                       code.data_ptr(), term.data_ptr(), 1e-9, ws.data_ptr(), st)), 4 * e * 2 + e),
        "vgg_post_partial": (lambda: L.check(lib.read_vgg_post_partial(raw.data_ptr(), m8.data_ptr(), n, H, W, C, bias.data_ptr(),
                                                                       nxt.data_ptr(), code.data_ptr(), term.data_ptr(), 1e-9,
                                                                       ws.data_ptr(), st)), 4 * e * 2 + e + p),
        "vgg_dgrad_in": (lambda: L.check(lib.read_vgg_dgrad_in(up.data_ptr(), 0, code.data_ptr(), n, H, W, C, g1.data_ptr(), 1e-9,
                                                               dy.data_ptr(), st)), e + 2 * e * 2),
        "vgg_dgrad_in_partial": (lambda: L.check(lib.read_vgg_dgrad_in_partial(up.data_ptr(), m8.data_ptr(), code.data_ptr(), n, H,
                                                                               W, C, g1.data_ptr(), 1e-9, dy.data_ptr(), st)),
                                 e + 2 * e * 2 + p),
        "vgg_image_grad": (lambda: L.check(lib.read_vgg_image_grad(x8.data_ptr(), n, H, W, std.data_ptr(), grad.data_ptr(), st)),
                           p * (16 + 12)),
        "vgg_image_grad_masked": (lambda: L.check(lib.read_vgg_image_grad_masked(x8.data_ptr(), m8.data_ptr(), n, H, W,
                                                                                 std.data_ptr(), grad.data_ptr(), st)),
                                  p * (16 + 12) + p),
    }
    t = {k: [] for k in arms}
    for _ in range(3):
        for k, (fn, _) in arms.items():
            t[k].append(timed(fn, reps))
    return {k: {"us": round(1e3 * float(np.median(t[k])), 2), "bytes": b,
                "hbm_share": round(b / HBM / (float(np.median(t[k])) * 1e-3), 3)} for k, (_, b) in arms.items()}


if __name__ == "__main__":
    main()
