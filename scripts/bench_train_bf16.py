"""C5 training step (8 crops of 256x256 per step, 5M points, L1 loss, backward through the net and the descriptor gather, Adam on
the net, sparse RMSprop on the descriptors) with the net trained in fp32 (torch operators, cuDNN), in bf16 (the 78 gated 3x3
stride-1 convs on the wgmma kernels, UNet.train_precision = 'bf16') and in bf16_all (all 99 convs), alternating in one process
so that clock drift hits all alike.
   python scripts/bench_train_bf16.py [--steps 10] [--rounds 3] [--batchnorm running|batch] [--out result.json]
--batchnorm batch puts the model in train() (the reference's default training: train-mode BatchNorm with batch statistics, and
NetAndTexture's per-item loop, B = 1 per net call) and then reports, instead of the eval-mode sections below, the step time per
precision, the time and bytes of the batch-statistics kernels at the C5 shapes, and the kernel launches per step with and without
the packed-filter cache (read_b200/blocks.py).  The default, running, is the eval-mode measurement:
Prints the card's name and power limit, per precision the step time and the share of the net's forward + backward in it, the time
to re-pack the 64 block convs' filters (done on every bf16 step), per stack shape the time of each backward kernel, the same for
the new shapes of the 14 single gated 3x3 convs (8-channel inputs, the RGB conv padded to C = 16) with the 8-channel input gradient
timed against the alternative of zero-padding the input and filters to 32 channels, and the forward + backward time of those 14
convs at their C5 shapes in each precision; then for the 21 1x1 / stride-2 convs of 'bf16_all' their forward + backward time at
C5 in fp32 and in bf16_all, per conv the time of each backward piece (RAW recompute, gate backward, weight gradient, input
gradient), and the activation bytes each precision saves for their backward."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from read_b200 import synth, ops, blocks, _lib as L, train as rtrain          # noqa: E402
from read_b200.unet import UNet                                                # noqa: E402
from read_b200.texture import PointTexture                                     # noqa: E402
from read_b200.compose import NetAndTexture                                    # noqa: E402

N, W, H, BC, LEVELS = 5_000_000, 256, 256, 8, 4


def ev():
    return torch.cuda.Event(enable_timing=True)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q}


def make_model(sd, tp, dev, batch=False):
    tex = PointTexture(8, N, init_method='zeros')
    with torch.no_grad():
        tex.texture_.copy_(torch.rand((1, 8, N), generator=torch.Generator().manual_seed(synth.SEED)))
    net = UNet()
    net.load_state_dict(sd, strict=True)
    net.train_precision = tp
    model = NetAndTexture(net, {0: tex}, 1)
    model.load_textures(0)
    model.to(dev)
    model.train(batch)                          # running: eval-mode BatchNorm (eval_in_train); batch: the reference's default
    return dict(net=net, tex=tex, model=model, opt_net=torch.optim.Adam(net.parameters(), lr=1e-4),
                opt_tex=rtrain.SparseRMSprop(tex, lr=1e-1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batchnorm", choices=("running", "batch"), default="running")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    batch = args.batchnorm == "batch"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    L.require_device(0)
    xyz = torch.from_numpy(synth.street_scene(N)).to(dev)
    store = ops.SortedPoints(xyz)
    pyr = ops.Pyramid(BC, W, H, LEVELS, dev)
    rng = np.random.default_rng(synth.SEED)
    n_mats = 3 + max(args.steps, 3)                 # 3 warm-up crops, then one per timed step and at least the 3 profiled ones
    mats = torch.stack([torch.from_numpy(synth.total_matrix(*synth.crop_cameras(W, H, rng.integers(0, 64, BC), rng)))
                        for _ in range(n_mats)]).to(dev)
    target = torch.rand((BC, 3, H, W), generator=torch.Generator().manual_seed(7)).to(dev)
    keys = ["uv_1d_p1"] + [f"uv_1d_p1_ds{l}" for l in range(1, LEVELS)]
    ids0 = torch.zeros(BC, dtype=torch.long)
    sd = synth.synth_state_dict(synth.SEED)
    runs = {tp: make_model(sd, tp, dev, batch) for tp in ("fp32", "bf16", "bf16_all")}

    def step(r, m, marks=None):
        e = [ev() for _ in range(4)] if marks is not None else None
        if e: e[0].record()
        pyr.clear()
        ops.raster_project_sorted(pyr, store, m)
        ops.raster_derive(pyr)
        inputs = {k: ops.zbuf_resolve(pyr, l, want_depth=False)[0].unsqueeze(1) for l, k in enumerate(keys)}
        inputs["id"] = ids0
        if e: e[1].record()
        loss = F.l1_loss(r["model"](inputs), target)
        loss.backward()
        if e: e[2].record()
        r["opt_net"].step()
        r["opt_tex"].step()
        r["opt_net"].zero_grad(set_to_none=True)
        if marks is not None:
            e[3].record()
            marks.append(e)
        return loss

    first_loss = {}
    for tp, r in runs.items():                     # warm-up (and the loss of both precisions on the same first crops)
        first_loss[tp] = float(step(r, mats[0]).detach())
        for s in range(1, 3):
            step(r, mats[s])
    torch.cuda.synchronize()
    ms = {tp: [] for tp in runs}
    share = {tp: [] for tp in runs}
    for _ in range(args.rounds):
        for tp, r in runs.items():
            torch.cuda.synchronize()
            a, b = ev(), ev()
            a.record()
            for s in range(args.steps):
                step(r, mats[3 + s])
            b.record()
            torch.cuda.synchronize()
            ms[tp].append(a.elapsed_time(b) / args.steps)
            marks = []
            for s in range(3):
                step(r, mats[3 + s], marks)
            torch.cuda.synchronize()
            net_ms = sum(e[1].elapsed_time(e[2]) for e in marks) / len(marks)
            tot_ms = sum(e[0].elapsed_time(e[3]) for e in marks) / len(marks)
            share[tp].append({"net_fwd_bwd_ms": net_ms, "step_ms": tot_ms, "share": net_ms / tot_ms})

    if batch:
        return report_batch(args, runs, ms, share, first_loss, step, mats, dev)

    # filter re-packing of the 64 block convs (what every bf16 step does before its first block launch)
    net = runs["bf16"]["net"]
    mods = [m for p in [f"Encoder.{i}" for i in range(4)] + [f"Decoder.{i}" for i in range(4)] for m in blocks.stack_convs(net, p)]
    pack = []
    for _ in range(5):
        a, b = ev(), ev()
        a.record()
        for m in mods:
            blocks.FoldedConv(m, *blocks.stack_params([m]))
        b.record()
        torch.cuda.synchronize()
        pack.append(a.elapsed_time(b))

    # backward kernels of one conv per stack shape at C5 (B = 8): RAW recompute, gate backward, weight gradient, input gradient
    lib = L.load()
    kern = []
    for C, S in ((32, 256), (64, 128), (128, 64), (256, 32)):
        m = next(mm for mm in mods if mm.block['conv_f'].weight.shape[0] == C)
        fc = blocks.FoldedConv(m, *blocks.stack_params([m]))
        x = torch.randn((BC, S, S, C), device=dev).bfloat16()
        dy = torch.randn((BC, S, S, C), device=dev).bfloat16()
        fm = torch.empty((BC, S, S, 2 * C), device=dev, dtype=torch.bfloat16)
        dfm = torch.empty_like(fm)
        red = torch.zeros((4, C), device=dev)
        dwf, dwm = torch.zeros_like(fc.wf), torch.zeros_like(fc.wm)
        st = L.stream_ptr()
        P = BC * S * S
        fns = {
            "raw_recompute": lambda: blocks._launch(lib, x, C, fc.w_tc, fc.par, fc.elu, L.OUT_RAW_NHWC, fm),
            "gate_backward": lambda: L.check(lib.read_gate_backward(dy.data_ptr(), fm.data_ptr(), P, C, 1, fc.bf.data_ptr(), fc.bm.data_ptr(),
                                                                    fc.scale.data_ptr(), fc.mean.data_ptr(), fc.inv.data_ptr(), dfm.data_ptr(),
                                                                    red[0].data_ptr(), red[1].data_ptr(), red[2].data_ptr(), red[3].data_ptr(), st)),
            "wgrad": lambda: L.check(lib.read_conv3x3_wgrad(dfm.data_ptr(), x.data_ptr(), BC, S, S, C, C, dwf.data_ptr(), dwm.data_ptr(), st)),
            "dgrad": lambda: blocks.dgrad(dfm, fc, residual=dy),
        }
        row = {"C": C, "HxW": f"{S}x{S}", "B": BC}
        for name, fn in fns.items():
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            a, b = ev(), ev()
            a.record()
            for _ in range(20):
                fn()
            b.record()
            torch.cuda.synchronize()
            row[name + "_us"] = a.elapsed_time(b) / 20 * 1e3
        flops = 2.0 * 2 * C * 9 * C * P
        row["wgrad_tflops"] = flops / (row["wgrad_us"] * 1e-6) / 1e12
        row["wgrad_min_bytes"] = P * 3 * C * 2            # [df | dm] and x read once
        row["wgrad_gbs"] = row["wgrad_min_bytes"] / (row["wgrad_us"] * 1e-6) / 1e9
        kern.append(row)

    # the new shapes of the 14 single convs at C5: (layer, Cin, C as launched, ELU, resolution)
    single = []
    for name, cin, C, elu, S in (("feat_extract.0", 8, 32, True, 256), ("feat_extract.5", 32, 16, False, 256),
                                 ("SCM2.main.0", 8, 16, True, 128), ("SCM1.main.0", 8, 32, True, 64), ("SCM0.main.0", 8, 64, True, 32)):
        m = net.get_submodule(name)
        fc = blocks.FoldedConv(m, *blocks.stack_params([m]), cout=C)
        x = torch.rand((BC, S, S, cin), device=dev).bfloat16()
        dy = torch.randn((BC, S, S, C), device=dev).bfloat16()
        fm = torch.empty((BC, S, S, 2 * C), device=dev, dtype=torch.bfloat16)
        dfm = torch.randn((BC, S, S, 2 * C), device=dev).bfloat16()
        red = torch.zeros((4, C), device=dev)
        dwf, dwm = torch.zeros_like(fc.wf), torch.zeros_like(fc.wm)
        st = L.stream_ptr()
        P = BC * S * S
        fns = {
            "raw_recompute": lambda: blocks._launch(lib, x, C, fc.w_tc, fc.par, fc.elu, L.OUT_RAW_NHWC, fm),
            "gate_backward": lambda: L.check(lib.read_gate_backward(dy.data_ptr(), fm.data_ptr(), P, C, int(elu), fc.bf.data_ptr(),
                                                                    fc.bm.data_ptr(), fc.scale.data_ptr(), fc.mean.data_ptr(),
                                                                    fc.inv.data_ptr(), dfm.data_ptr(), red[0].data_ptr(),
                                                                    red[1].data_ptr(), red[2].data_ptr(), red[3].data_ptr(), st)),
            "wgrad": lambda: L.check(lib.read_conv3x3_wgrad(dfm.data_ptr(), x.data_ptr(), BC, S, S, C, cin, dwf.data_ptr(),
                                                            dwm.data_ptr(), st)),
            "dgrad": lambda: blocks.dgrad(dfm, fc),
        }
        if cin == 8:
            # the alternative: the input and the filters zero-padded to 32 channels, the TMA kernel's RAW dgrad (N = 32), and
            # the padded input's copy that the weight gradient would then read
            zpad = lambda t: torch.cat([t, t.new_zeros(t.shape[:1] + (24,) + t.shape[2:])], 1)
            fc32 = blocks.FoldedConv(m, zpad(m.block['conv_f'].weight), m.block['conv_f'].bias, zpad(m.block['conv_m'].weight),
                                     m.block['conv_m'].bias, m.block['norm'].weight, m.block['norm'].bias, cout=C)
            fns["dgrad_padded32"] = lambda: blocks.dgrad(dfm, fc32)
            fns["pad_input_to_32"] = lambda: F.pad(x, (0, 24))
        row = {"layer": name, "Cin": cin, "C": C, "HxW": f"{S}x{S}", "B": BC}
        for kname, fn in fns.items():
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            a, b = ev(), ev()
            a.record()
            for _ in range(20):
                fn()
            b.record()
            torch.cuda.synchronize()
            row[kname + "_us"] = a.elapsed_time(b) / 20 * 1e3
        single.append(row)

    # forward + backward of the 14 single convs at their C5 shapes, fp32 (torch / cuDNN) against bf16 (GatedConvFn)
    shapes = [("feat_extract.0", 256), ("feat_extract.5", 256)] + \
             [(f"SCM{i}.main.{j}", 32 << i) for i in range(3) for j in (0, 2)] + \
             [(f"AFFs.{i}.conv.1", 256 >> i) for i in range(3)] + [(f"FAM{i}.merge", 32 << i) for i in range(3)]
    assert len(shapes) == 14
    singles_ms = {}
    for tp in ("fp32", "bf16"):
        case = []
        for name, S in shapes:
            m = runs[tp]["net"].get_submodule(name)
            cin = m.block['conv_f'].weight.shape[1]
            x = torch.rand((BC, cin, S, S), device=dev, requires_grad=True)
            gy = torch.randn((BC, m.block['conv_f'].weight.shape[0], S, S), device=dev)
            case.append((m, x, gy))

        def run_all():
            for m, x, gy in case:
                y = blocks.gated_conv(m, x) if tp == "bf16" else m(x)
                y.backward(gy)
        for _ in range(3):
            run_all()
        torch.cuda.synchronize()
        vals = []
        for _ in range(args.rounds):
            a, b = ev(), ev()
            a.record()
            for _ in range(5):
                run_all()
            b.record()
            torch.cuda.synchronize()
            vals.append(a.elapsed_time(b) / 5)
        singles_ms[tp] = vals
    for tp in runs:
        runs[tp]["opt_net"].zero_grad(set_to_none=True)

    # the 21 1x1 / stride-2 convs at C5: (layer, sources' (channels, resolution)); forward + backward in fp32 (torch, the concat
    # on torch) against bf16_all (MultiSourceConvFn, a virtual concat), and per conv the backward's pieces
    new_convs = [("feat_extract.1", [(32, 256)]), ("feat_extract.2", [(64, 128)]), ("feat_extract.6", [(128, 64)]),
                 ("feat_extract.7", [(256, 32)]), ("feat_extract.3", [(128, 64)]), ("feat_extract.4", [(64, 128)]),
                 ("Convs.0", [(128, 64)] * 2), ("Convs.1", [(64, 128)] * 2), ("Convs.2", [(32, 256)] * 2)] + \
                [(f"AFFs.{i}.conv.0", [(c, 256 >> i) for c in (32, 64, 128, 256)]) for i in range(3)] + \
                [(f"SCM{i}.{n}", [(c << (2 - i), 32 << i)]) for i in range(3) for n, c in (("main.1", 16), ("main.3", 32), ("conv", 64))]
    assert len(new_convs) == 21
    saved_bytes = {"fp32_conv_inputs": 0, "bf16_all_sources": 0}
    new_ms, new_kern = {}, []
    for tp in ("fp32", "bf16_all"):
        case = []
        for name, srcs in new_convs:
            m = runs[tp]["net"].get_submodule(name)
            xs = [torch.rand((BC, c, S, S), device=dev, requires_grad=True) for c, S in srcs]
            S = srcs[0][1] // m.stride
            gy = torch.randn((BC, m.block['conv_f'].weight.shape[0], S, S), device=dev)
            case.append((name, m, xs, gy))
            if tp == "fp32":
                saved_bytes["fp32_conv_inputs"] += sum(x.numel() for x in xs) * 4
                saved_bytes["bf16_all_sources"] += sum(x.numel() for x in xs) * 2

        def run_all():
            for name, m, xs, gy in case:
                y = blocks.gated_conv_srcs(m, xs, name) if tp == "bf16_all" else m(torch.cat(xs, 1) if len(xs) > 1 else xs[0])
                y.backward(gy)
        for _ in range(3):
            run_all()
        torch.cuda.synchronize()
        vals = []
        for _ in range(args.rounds):
            a, b = ev(), ev()
            a.record()
            for _ in range(5):
                run_all()
            b.record()
            torch.cuda.synchronize()
            vals.append(a.elapsed_time(b) / 5)
        new_ms[tp] = vals
        if tp != "bf16_all":
            continue
        for name, m, xs, gy in case:
            ts = [ops.nchw_to_nhwc(x.detach(), True) for x in xs]
            C = blocks.padded_channels(m.block['conv_f'].weight.shape[0])
            fc = blocks.FoldedConv(m, *blocks.stack_params([m]), cout=C, srcs=ts)
            fm = blocks.recompute_fm(lib, ts, fc)
            B_, Ho, Wo, _ = fm.shape
            Hi, Wi = ts[0].shape[1:3]
            dy = torch.randn((B_, Ho, Wo, C), device=dev).bfloat16()
            dfm = torch.randn_like(fm)
            red = torch.zeros((4, C), device=dev)
            dwf, dwm = torch.zeros_like(fc.wf), torch.zeros_like(fc.wm)
            st = L.stream_ptr()
            P = B_ * Ho * Wo

            def wgrad():
                for t in ts:
                    L.check(lib.read_conv_wgrad(dfm.data_ptr(), t.data_ptr(), B_, Hi, Wi, Ho, Wo, C, t.shape[3], fc.k, fc.stride,
                                                dwf.data_ptr(), dwm.data_ptr(), st))

            def dgrad():
                if fc.stride == 2:
                    dx = torch.empty_like(ts[0])
                    L.check(lib.read_conv_dgrad_s2(dfm.data_ptr(), blocks.dgrad_s2_filters(fc).data_ptr(), B_, Ho, Wo, C,
                                                   ts[0].shape[3], fc.k, dx.data_ptr(), st))
                    return
                c0 = 0
                for t in ts:
                    blocks.dgrad_1x1(dfm, fc, c0, t.shape[3])
                    c0 += t.shape[3]
            fns = {
                "raw_recompute": lambda: blocks.recompute_fm(lib, ts, fc),
                "gate_backward": lambda: L.check(lib.read_gate_backward(dy.data_ptr(), fm.data_ptr(), P, C, int(fc.elu), fc.bf.data_ptr(),
                                                                        fc.bm.data_ptr(), fc.scale.data_ptr(), fc.mean.data_ptr(),
                                                                        fc.inv.data_ptr(), dfm.data_ptr(), red[0].data_ptr(),
                                                                        red[1].data_ptr(), red[2].data_ptr(), red[3].data_ptr(), st)),
                "wgrad": wgrad,
                "dgrad": dgrad,
            }
            row = {"layer": name, "sources": [t.shape[3] for t in ts], "C": C, "k": fc.k, "stride": fc.stride,
                   "in": f"{Hi}x{Wi}", "out": f"{Ho}x{Wo}", "B": BC}
            for kname, fn in fns.items():
                for _ in range(3):
                    fn()
                torch.cuda.synchronize()
                a, b = ev(), ev()
                a.record()
                for _ in range(20):
                    fn()
                b.record()
                torch.cuda.synchronize()
                row[kname + "_us"] = a.elapsed_time(b) / 20 * 1e3
            flops = 2.0 * 2 * C * fc.k * fc.k * sum(t.shape[3] for t in ts) * P     # one GEMM of the conv pair
            row["wgrad_tflops"] = flops / (row["wgrad_us"] * 1e-6) / 1e12
            row["dgrad_tflops"] = flops / (row["dgrad_us"] * 1e-6) / 1e12
            new_kern.append(row)
    for tp in runs:
        runs[tp]["opt_net"].zero_grad(set_to_none=True)

    res = {"card": card(), "steps": args.steps, "rounds": args.rounds, "crops_per_step": BC, "size": f"{W}x{H}", "n_points": N,
           "ms_per_step": ms, "net_fwd_bwd_per_step": share, "first_loss": first_loss,
           "bf16_filter_repack_ms_per_step": pack, "backward_kernels": kern, "single_conv_kernels": single,
           "single_convs_fwd_bwd_ms_per_step": singles_ms, "new_convs_fwd_bwd_ms_per_step": new_ms, "new_conv_kernels": new_kern,
           "new_convs_saved_bytes_per_step": saved_bytes}
    for tp in runs:
        med = sorted(ms[tp])[len(ms[tp]) // 2]
        sh = sorted(share[tp], key=lambda x: x["share"])[len(share[tp]) // 2]
        print(f"{tp}: {med:.2f} ms/step (rounds {', '.join(f'{v:.2f}' for v in ms[tp])}), net fwd+bwd {sh['net_fwd_bwd_ms']:.2f} ms "
              f"of a {sh['step_ms']:.2f} ms profiled step = {100 * sh['share']:.1f} %")
    print(f"card: {res['card']}")
    print(f"first-step loss fp32 {first_loss['fp32']:.6f} bf16 {first_loss['bf16']:.6f} bf16_all {first_loss['bf16_all']:.6f}; "
          f"filter re-pack {sorted(pack)[2]:.3f} ms/step")
    for row in kern + single + new_kern:
        print(json.dumps(row))
    for tp, v in singles_ms.items():
        print(f"14 single 3x3 convs fwd+bwd at C5, {tp}: {sorted(v)[len(v) // 2]:.2f} ms/step (rounds {', '.join(f'{x:.2f}' for x in v)})")
    for tp, v in new_ms.items():
        print(f"21 1x1 / stride-2 convs fwd+bwd at C5, {tp}: {sorted(v)[len(v) // 2]:.2f} ms/step (rounds {', '.join(f'{x:.2f}' for x in v)})")
    print(f"activations saved for the 21 convs' backward at C5: {saved_bytes}")
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        json.dump(res, open(args.out, "w"), indent=1)


def report_batch(args, runs, ms, share, first_loss, step, mats, dev):
    """--batchnorm batch: step times, the batch-statistics kernels at the C5 shapes (one net call = one 256x256 crop, so the
    stacks run at P = 65536 / 16384 / 4096 / 1024 pixels with C = 32 / 64 / 128 / 256) and the launches per step."""
    lib = L.load()
    launches = {}
    for tp in ("bf16", "bf16_all"):
        for cached in (True, False):
            blocks.cache_filters = cached
            blocks.clear_filter_cache()
            step(runs[tp], mats[-1])                                          # fills the cache (or not)
            torch.cuda.synchronize()
            n0 = ops.launch_count()
            step(runs[tp], mats[-2])
            torch.cuda.synchronize()
            launches[f"{tp}, filter cache {'on' if cached else 'off'}"] = ops.launch_count() - n0
    blocks.cache_filters = True
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    step(runs["fp32"], mats[-1])
    torch.cuda.synchronize()
    launches["fp32 (library kernels only: raster, gather, descriptors)"] = ops.launch_count() - n0

    kern = []
    reps = 50
    for C, side in ((32, 256), (64, 128), (128, 64), (256, 32)):
        P = side * side
        g = torch.randn((P, C), device=dev).bfloat16()
        fm = torch.randn((P, 2 * C), device=dev).bfloat16()
        dy = torch.randn((P, C), device=dev).bfloat16()
        dfm, y = torch.empty_like(fm), torch.empty_like(g)
        v = torch.rand((10, C), device=dev) + 0.5
        red = torch.zeros((4, C), device=dev)
        ws = torch.empty(lib.read_bn_workspace_bytes(C), dtype=torch.uint8, device=dev)
        st = L.stream_ptr()
        p = [t.data_ptr() for t in v]
        fns = {
            "bn_stats": (lambda: L.check(lib.read_bn_batch_stats(g.data_ptr(), P, C, C, p[0], p[1], 1e-5, 0.1, p[2], p[3], p[4],
                                                                 p[5], None, p[6], p[7], ws.data_ptr(), st)), P * C * 2),
            "bn_apply": (lambda: L.check(lib.read_bn_apply(g.data_ptr(), P, C, p[6], p[7], None, y.data_ptr(), st)), 2 * P * C * 2),
            "bn_backward_reduce": (lambda: L.check(lib.read_bn_backward_reduce(dy.data_ptr(), fm.data_ptr(), P, C, 1, p[0], p[1],
                                                                               p[4], p[5], red[3].data_ptr(), red[2].data_ptr(),
                                                                               st)), 3 * P * C * 2),
            "gate_backward_batch_stats": (lambda: L.check(lib.read_gate_backward_batch_stats(
                dy.data_ptr(), fm.data_ptr(), P, C, 1, p[0], p[1], p[6], p[4], p[5], red[3].data_ptr(), red[2].data_ptr(),
                dfm.data_ptr(), red[0].data_ptr(), red[1].data_ptr(), st)), 5 * P * C * 2),
        }
        for name, (fn, nbytes) in fns.items():
            for _ in range(5):
                fn()
            rounds = []
            for _ in range(3):
                a, b = ev(), ev()
                a.record()
                for _ in range(reps):
                    fn()
                b.record()
                torch.cuda.synchronize()
                rounds.append(a.elapsed_time(b) * 1e3 / reps)
            us = sorted(rounds)[1]
            kern.append({"kernel": name, "C": C, "pixels": P, "us": round(us, 2), "rounds_us": [round(x, 2) for x in rounds],
                         "bytes": nbytes, "share_of_3.35TB/s": round(nbytes / (us * 1e-6) / 3.35e12, 3)})

    res = {"card": card(), "batchnorm": "batch", "steps": args.steps, "rounds": args.rounds, "crops_per_step": BC,
           "size": f"{W}x{H}", "n_points": N, "ms_per_step": ms, "net_fwd_bwd_per_step": share, "first_loss": first_loss,
           "launches_per_step": launches, "batch_stats_kernels": kern}
    print(f"card: {res['card']}")
    for tp in runs:
        med = sorted(ms[tp])[len(ms[tp]) // 2]
        sh = sorted(share[tp], key=lambda x: x["share"])[len(share[tp]) // 2]
        print(f"{tp} (train mode): {med:.2f} ms/step (rounds {', '.join(f'{v:.2f}' for v in ms[tp])}), net fwd+bwd "
              f"{sh['net_fwd_bwd_ms']:.2f} ms of a {sh['step_ms']:.2f} ms profiled step")
    print("first-step loss " + ", ".join(f"{tp} {v:.6f}" for tp, v in first_loss.items()))
    for k, v in launches.items():
        print(f"library kernel launches per step, {k}: {v}")
    for row in kern:
        print(json.dumps(row))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        json.dump(res, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
