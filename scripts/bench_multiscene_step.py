"""The reference's headless training step (tests/headless_util.train_step: MyRender -> ModelAndLoss -> vgg + 1e4 * huber -> Adam and
SparseRMSprop) at bf16_all with read_b200.vgg_loss.VGGLoss, over 2 and 4 synthetic scenes of 5M points.  Each batch is 2 samples x
4 crops of 256x256, from two different scenes.  Arms, alternated over the rounds in one process, each in eval mode (eval_in_train)
and in train() with per-item BatchNorm:
  loop      the per-crop loop (NetAndTexture's dispatch patched here to refuse the multi-texture table): 8 net calls per step;
  batched   the same mixed batches in one net call, the items gathering from their own textures;
  one-scene batches whose 8 crops all come from one scene: the one-texture batched call.
Also times the multi-texture gather forward and sparse backward at the step's level-0 shape against the single-texture kernels, on
index maps rendered from the scenes.
   python scripts/bench_multiscene_step.py [--steps 10] [--rounds 3] [--out result.json]
Prints the card's name and power limit, per arm the step time of each round (CUDA events over --steps steps, after 3 warm-up steps)
and the library's kernel launches per step; per kernel the time (CUDA events over 50 calls) and its share of 3.35 TB/s."""
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
from read_b200 import headless, ops, synth, _lib as L             # noqa: E402
from read_b200.myrender import MyRender                           # noqa: E402
from read_b200.vgg_loss import VGGLoss                            # noqa: E402
from bench_train_bf16 import card, ev, N, W, H, BC                # noqa: E402
import headless_util as hu                                        # noqa: E402
import vgg_util                                                   # noqa: E402

WARMUP = 3
HBM = 3.35e12                     # H100 SXM data sheet, bytes/s
VARIANTS = ("loop", "batched", "one-scene")
MODES = ("eval", "train per_item")


def make_pipeline(scenes, mode, sd):
    for name in ("READ", "READ.datasets", "READ.datasets.dynamic"):
        sys.modules[name] = hu.datasets_module(scenes, [None] * len(scenes))
    p = headless.TexturePipeline()
    p.create(hu.pipeline_args(net_train_precision="bf16_all", net_train_batchnorm='per_item' if mode != "eval" else 'batch',
                              criterion_module=VGGLoss, criterion_args={'features': vgg_util.seeded_features()}))
    p.net.load_state_dict(sd, strict=True)
    with torch.no_grad():
        for i, t in p.textures.items():
            t.texture_.copy_(torch.rand((1, 8, N), generator=torch.Generator().manual_seed(synth.SEED + i)))
    p.model.train(mode != "eval")
    p.dataset_load(scenes)
    extra = p.extra_optimizer(scenes)
    p.model.cuda()
    return dict(pipeline=p, extra=extra, model=hu.ModelAndLoss(p.model, p.criterion))


def crops(pair, seed):
    """2 samples x 4 crops: scene pair[0]'s, then pair[1]'s."""
    rng = np.random.default_rng(seed)
    halves = [hu.batch(W, H, rng.integers(0, 64, BC // 2), ds_id=s, seed=seed * 2 + k) for k, s in enumerate(pair)]
    return {'input': {'id': torch.cat([h['input']['id'] for h in halves])},
            'proj_matrix': torch.cat([h['proj_matrix'] for h in halves]), 'view_matrix': torch.cat([h['view_matrix'] for h in halves])}


def batches(n_scenes, variant, count):
    out = []
    for s in range(count):
        a = s % n_scenes
        pair = (a, a) if variant == "one-scene" else (a, (a + 1 + (s // n_scenes) % (n_scenes - 1)) % n_scenes)
        out.append(crops(pair, s))
    return out


def run(arm, variant, renderer, data, target, dev):
    p, model = arm["pipeline"], arm["pipeline"].model
    if variant == "loop":
        model._texture_table = lambda texture_ids: None          # the parent's dispatch: every mixed batch takes the loop
    try:
        for d in data:
            hu.train_step(renderer, arm["model"], d, target, None, dev, p, arm["extra"])
    finally:
        model.__dict__.pop("_texture_table", None)


def time_kernels(renderer, scene_pair_batch, textures, dev):
    """The multi-texture gather (forward, NCHW f32) and sparse backward at the step's level 0, against the single-texture kernels on
    the same index map with one texture."""
    inputs, _ = renderer.render(scene_pair_batch)
    key = hu.INPUT_FORMAT.replace(' ', '').split(',')[0]
    ids = inputs[key][:, 0].to(dev).contiguous()
    slots = [0] * (BC // 2) + [1] * (BC // 2)
    nds = [t.point_major() for t in textures]
    B_, h, w = ids.shape
    px = B_ * h * w
    nonempty = int((ids != 0).sum())
    go = torch.rand((B_, 8, h, w), device=dev)
    acc = [torch.zeros((N, 8), device=dev) for _ in range(2)]
    flags = [torch.zeros(N, dtype=torch.uint8, device=dev) for _ in range(2)]
    out = torch.empty((B_, 8, h, w), device=dev)
    lib, sp = L.load(), L.stream_ptr()
    calls = {
        "gather items": lambda: ops.gather_from_index_items(nds, slots, ids, L.FEAT_NCHW_F32, out=out),
        "gather single": lambda: ops.gather_from_index(nds[0], ids, L.FEAT_NCHW_F32, out=out),
        "sparse backward items": lambda: ops.gather_backward_items(go, ids, slots, [N, N], acc, flags),
        "sparse backward single": lambda: L.check(lib.read_gather_backward_sparse(go.data_ptr(), ids.data_ptr(), B_, 8, h, w, N,
                                                                                  acc[0].data_ptr(), flags[0].data_ptr(), sp)),
    }
    # bytes each must move: ids (4 B) and the feature / gradient map (32 B) per pixel, plus one 32-byte descriptor row read per pixel
    # (forward) or one 32-byte accumulator row read and written per non-empty pixel and its touched byte (backward)
    nbytes = {"gather": px * (4 + 32 + 32), "sparse backward": px * (4 + 32) + nonempty * (64 + 1)}
    res = {}
    for name, fn in calls.items():
        for _ in range(5):
            fn()
        a, b = ev(), ev()
        a.record()
        for _ in range(50):
            fn()
        b.record()
        torch.cuda.synchronize()
        us = a.elapsed_time(b) * 1e3 / 50
        nb = nbytes[name.rsplit(' ', 1)[0]]
        res[name] = {"us": us, "bytes": nb, "share_of_hbm": nb / (us * 1e-6) / HBM}
    return res, {"shape": [B_, h, w], "nonempty_pixels": nonempty}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    L.require_device(0)
    scenes = [hu.scene(N, W, H, name=f"scene{i}", ds_id=i, seed=synth.SEED + i, depth=250.0) for i in range(4)]
    renderer = MyRender()
    renderer.update_ds(scenes)
    target = torch.rand((BC, 3, H, W), generator=torch.Generator().manual_seed(7)).to(dev)
    sd = synth.synth_state_dict(synth.SEED)
    out = {"card": card(), "shape": f"{BC} crops of {W}x{H} (2 samples x 4 crops), {N} points per scene, "
                                    f"{len(hu.INPUT_FORMAT.split(','))} levels, bf16_all + VGGLoss",
           "step_ms": {}, "step_ms_median": {}, "launches_per_step": {}}
    print(json.dumps(out["card"]), flush=True)
    for n_scenes in (2, 4):
        for mode in MODES:
            arm = make_pipeline(scenes[:n_scenes], mode, sd)
            data = {v: batches(n_scenes, v, WARMUP + args.steps) for v in VARIANTS}
            for v in VARIANTS:
                run(arm, v, renderer, data[v][:WARMUP], target, dev)
            torch.cuda.synchronize()
            for v in VARIANTS:
                name = f"{n_scenes} scenes, {mode}, {v}"
                out["step_ms"][name] = []
                n0 = ops.launch_count()
                run(arm, v, renderer, data[v][:1], target, dev)
                torch.cuda.synchronize()
                out["launches_per_step"][name] = ops.launch_count() - n0
            for _ in range(args.rounds):
                for v in VARIANTS:
                    a, b = ev(), ev()
                    a.record()
                    run(arm, v, renderer, data[v][WARMUP:], target, dev)
                    b.record()
                    torch.cuda.synchronize()
                    out["step_ms"][f"{n_scenes} scenes, {mode}, {v}"].append(a.elapsed_time(b) / args.steps)
            for v in VARIANTS:
                name = f"{n_scenes} scenes, {mode}, {v}"
                out["step_ms_median"][name] = float(np.median(out["step_ms"][name]))
                print(f"{name:36s} step " + ", ".join(f"{t:.1f}" for t in out["step_ms"][name]) +
                      f" ms (median {out['step_ms_median'][name]:.1f}), {out['launches_per_step'][name]} library launches per step",
                      flush=True)
            if n_scenes == 2 and mode == "eval":
                textures = [arm["pipeline"].textures[i] for i in range(2)]
                out["kernels"], out["kernel_shape"] = time_kernels(renderer, crops((0, 1), 999), textures, dev)
            del arm
            torch.cuda.empty_cache()
    print(f"kernels at {out['kernel_shape']}:")
    for name, r in out["kernels"].items():
        print(f"  {name:24s} {r['us']:8.1f} us, {r['bytes'] / 1e6:.1f} MB, {100 * r['share_of_hbm']:.1f} % of 3.35 TB/s")
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
