"""A/B of whole C3 frames between two builds of the library, alternating bench.py processes, plus the per-layer times of the
3x3 stride-1 C -> C gated convs (bench.py --layer-times) and the max-abs difference of the two builds' dumped frames.

    python -m read_b200.build                                    # build B: the tree's library
    python scripts/bench_conv_c32.py --lib-a /path/to/other/libread_b200.so --rounds 5 --out /tmp/c32

Arm A loads --lib-a through READ_B200_LIB (e.g. a parent commit's library compiled elsewhere and copied next to the tree);
arm B loads the tree's own read_b200/libread_b200.so.  Rounds run A, B, A, B, ...  Prints one JSON summary (medians and
ranges of bench.py's value and e2e frames/s, per-class layer times and TFLOP/s) and writes it with every raw line to --out.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or q.stderr.strip()


def run_arm(lib, steps, warmup, out_dir, tag, dump):
    env = dict(os.environ)
    env.pop("READ_B200_LIB", None)
    if lib:
        env["READ_B200_LIB"] = os.path.abspath(lib)
    lt = os.path.join(out_dir, f"layers_{tag}.json")
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(steps), "--warmup", str(warmup),
           "--layer-times", lt]
    if dump:
        cmd += ["--dump-outputs", os.path.join(out_dir, f"frame_{tag}")]
    p = subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=ROOT)
    lines = [ln for ln in p.stdout.splitlines() if ln.startswith("{") and '"metric"' in ln]
    if p.returncode != 0 or not lines:
        raise RuntimeError(f"bench.py ({tag}) failed with {p.returncode}:\n{p.stderr[-3000:]}")
    res = json.loads(lines[-1])
    layers = json.load(open(lt))
    return res, layers


def stats(v):
    return {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v)), "n": len(v)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib-a", required=True, help="library of arm A (loaded through READ_B200_LIB)")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "bench_conv_c32"),
                    help="directory for the summary, the per-run layer times and the dumped frames")
    ap.add_argument("--names", default="Encoder.0.,Decoder.3.,AFFs.0.conv.1",
                    help="comma-separated layer-name prefixes of the class to report (default: the 32-channel 3x3 layers)")
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    info = {"gpu": gpu_info()}
    print(json.dumps(info), flush=True)
    prefixes = tuple(args.names.split(","))
    arms = {"A": args.lib_a, "B": None}
    vals = {k: {"value": [], "e2e": [], "class_ms": [], "parity_ok": []} for k in arms}
    per_layer = {k: {} for k in arms}
    raw = []
    for r in range(args.rounds):
        for k, lib in arms.items():
            res, layers = run_arm(lib, args.steps, args.warmup, args.out, f"{k}{r}", dump=r == 0)
            raw.append({"arm": k, "round": r, "result": res})
            v = vals[k]
            v["value"].append(res["value"])
            v["e2e"].append(res["e2e"]["value"])
            v["parity_ok"].append(bool(res["parity"] and res["parity"].get("ok")))
            sel = [row for row in layers if row["name"].startswith(prefixes) and row["impl"] >= 0 and row["gflop"] > 0]
            v["class_ms"].append(sum(row["ms"] for row in sel))
            for row in sel:
                per_layer[k].setdefault(row["name"], []).append((row["ms"], row["tflops"], row["gflop"]))
            print(json.dumps({"arm": k, "round": r, "value": res["value"], "e2e": res["e2e"]["value"],
                              "class_ms": v["class_ms"][-1], "layers": len(sel)}), flush=True)
    summary = dict(info)
    for k in arms:
        summary[k] = {"lib": arms[k] or "tree", "value_fps": stats(vals[k]["value"]), "e2e_fps": stats(vals[k]["e2e"]),
                      "class_ms_per_frame": stats(vals[k]["class_ms"]), "parity_ok": all(vals[k]["parity_ok"]),
                      "layers": {n: {"ms": float(np.median([x[0] for x in xs])), "tflops": float(np.median([x[1] for x in xs])),
                                     "gflop": xs[0][2]} for n, xs in sorted(per_layer[k].items())}}
    try:
        fa = np.load(os.path.join(args.out, "frame_A0", "frame.npy"))
        fb = np.load(os.path.join(args.out, "frame_B0", "frame.npy"))
        summary["frame_max_abs_diff"] = float(np.abs(fa.astype(np.float64) - fb).max())
    except OSError as e:
        summary["frame_max_abs_diff"] = f"unavailable: {e}"
    json.dump({"summary": summary, "raw": raw}, open(os.path.join(args.out, "summary.json"), "w"), indent=1)
    print(json.dumps(summary, indent=1), flush=True)


if __name__ == "__main__":
    main()
