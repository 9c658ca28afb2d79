"""The reference's headless training step (src/train.py --headless, restated in tests/headless_util.py) at C5: 8 crops of 256x256,
5M points, the example config's five 'uv' levels, vgg + 1e4 * huber, Adam on the net and the pipeline's sparse RMSprop on the
descriptors, the index maps coming back through the CPU as MyRender.render returns them.  The pipeline is
read_b200.headless.TexturePipeline, built through a stand-in for READ.datasets.dynamic.  Arms, alternated over the rounds in one
process:
  fp32      the net on torch operators with the VGG loss on torch (what the trainer runs with only pcpr / MyRender swapped in);
  bf16_all  every conv of the net and the VGG loss on our kernels (--net_train_precision bf16_all, read_b200.vgg_loss.VGGLoss);
each in eval mode (eval_in_train) and in train() with per-item BatchNorm (--net_train_batchnorm per_item).
   python scripts/bench_headless_step.py [--steps 10] [--rounds 3] [--out result.json]
Prints the card's name and power limit, per arm the step time of each round (CUDA events over --steps steps, after 3 warm-up
steps), and the share of the step between the events around MyRender.render + to_device (the index-map round trip)."""
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
from read_b200 import headless, synth, _lib as L                  # noqa: E402
from read_b200.myrender import MyRender                           # noqa: E402
from read_b200.vgg_loss import VGGLoss                            # noqa: E402
from bench_train_bf16 import card, ev, N, W, H, BC                # noqa: E402
import headless_util as hu                                        # noqa: E402
import vgg_util                                                   # noqa: E402

WARMUP = 3
ARMS = {f"{precision} {mode}": (precision, mode) for mode in ("eval", "train per_item") for precision in ("fp32", "bf16_all")}


def make_arm(precision, mode, scene, sd):
    crit = (hu.TorchVGG if precision == "fp32" else VGGLoss, {'features': vgg_util.seeded_features()})
    for name in ("READ", "READ.datasets", "READ.datasets.dynamic"):
        sys.modules[name] = hu.datasets_module([scene], [None])
    p = headless.TexturePipeline()
    p.create(hu.pipeline_args(net_train_precision=precision, net_train_batchnorm='per_item' if mode != "eval" else 'batch',
                              criterion_module=crit[0], criterion_args=crit[1]))
    p.net.load_state_dict(sd, strict=True)
    with torch.no_grad():
        p.textures[0].texture_.copy_(torch.rand((1, 8, N), generator=torch.Generator().manual_seed(synth.SEED)))
    p.model.train(mode != "eval")
    p.dataset_load([scene])
    extra = p.extra_optimizer([scene])
    p.model.cuda()
    return dict(pipeline=p, extra=extra, model=hu.ModelAndLoss(p.model, p.criterion))


def run(arm, renderer, batches, target, dev, times=None):
    """One step per batch; with ``times``, append per step the events before render, after to_device and after the step."""
    p = arm["pipeline"]
    for data in batches:
        a, b, c = ev(), ev(), ev()
        a.record()
        inputs, _ = renderer.render(data)
        data_input = hu.to_device(inputs, dev)
        b.record()
        output, loss_dict = arm["model"](data_input, target, label=None, mask=None)
        loss = hu.step_loss(output, loss_dict, None, p.model.reg_loss())
        loss.backward()
        p.optimizer.step()
        p.optimizer.zero_grad()
        arm["extra"].step()
        arm["extra"].zero_grad()
        c.record()
        if times is not None:
            times.append((a, b, c))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    L.require_device(0)
    scene = hu.scene(N, W, H, depth=250.0)
    renderer = MyRender()
    renderer.update_ds([scene])
    rng = np.random.default_rng(synth.SEED)
    batches = [hu.batch(W, H, rng.integers(0, 64, BC), seed=s) for s in range(WARMUP + args.steps)]
    target = torch.rand((BC, 3, H, W), generator=torch.Generator().manual_seed(7)).to(dev)
    sd = synth.synth_state_dict(synth.SEED)
    arms = {name: make_arm(precision, mode, scene, sd) for name, (precision, mode) in ARMS.items()}
    for arm in arms.values():
        run(arm, renderer, batches[:WARMUP], target, dev)
    torch.cuda.synchronize()
    step_ms = {name: [] for name in arms}
    share = {name: [] for name in arms}
    for _ in range(args.rounds):
        for name, arm in arms.items():
            times = []
            run(arm, renderer, batches[WARMUP:], target, dev, times)
            torch.cuda.synchronize()
            total = times[0][0].elapsed_time(times[-1][2])
            trip = sum(a.elapsed_time(b) for a, b, _ in times)
            step_ms[name].append(total / len(times))
            share[name].append(trip / total)
    out = {"card": card(), "shape": f"{BC} crops of {W}x{H}, {N} points, {len(hu.INPUT_FORMAT.split(','))} levels",
           "step_ms": step_ms, "step_ms_median": {k: float(np.median(v)) for k, v in step_ms.items()},
           "round_trip_share": share, "round_trip_share_median": {k: float(np.median(v)) for k, v in share.items()}}
    print(json.dumps(out["card"]))
    for name in arms:
        print(f"{name:20s} step " + ", ".join(f"{t:.2f}" for t in step_ms[name]) + f" ms (median {out['step_ms_median'][name]:.2f}),"
              f" index-map round trip {100 * out['round_trip_share_median'][name]:.1f} % of the step")
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
