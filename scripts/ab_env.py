"""ABAB of an engine-construction environment switch on whole-net CUDA-graph replays (C3 shapes) plus per-layer in-sequence times.
   python scripts/ab_env.py READ_B200_ALT_ORDER 0 1      |      python scripts/ab_env.py opt:tc_pdl 1 0"""
import os, sys
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from read_b200 import synth, _lib as L
from read_b200.engine import UNetEngine

VAR, VALS = sys.argv[1], sys.argv[2:]
dev = torch.device("cuda", 0)
sd = synth.synth_state_dict(synth.SEED)
H, W = 1088, 1920
g = torch.Generator().manual_seed(3)
feats = [torch.rand((1, 8, H >> l, W >> l), generator=g) for l in range(4)]


def mk(v):
    if VAR.startswith("opt:"):               # a read_set_option, e.g. opt:tc_pdl
        L.check(L.load().read_set_option(VAR[4:].encode(), int(v)))
    else:
        os.environ[VAR] = v
    e = UNetEngine(sd, 1, H, W, dev, precision="bf16", use_graph=True)
    e.set_inputs_nchw([f.to(dev) for f in feats])
    for _ in range(3):
        e.run()
    torch.cuda.synchronize()
    return e


def t1(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); fn(); b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b)


variants = [(f"{VAR}={v}", mk(v)) for v in VALS]
ref = variants[0][1].output.clone()
print({k: bool(torch.equal(e.output, ref)) for k, e in variants}, flush=True)
ts = {k: [] for k, _ in variants}
for rep in range(15):
    for k, e in variants:
        ts[k].append(t1(e.run))
print({k: round(float(np.median(v[3:])), 4) for k, v in ts.items()}, "ms per net replay")
