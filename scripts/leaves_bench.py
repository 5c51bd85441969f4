"""What handing out the leaves costs: ms per call of Pipeline.currentLeaves() / modelLeaves() (lists of host vectors),
currentLeavesArray() / modelLeavesArray() (numpy) and *Array(device=True) followed by a stream sync (CUDA tensors), on
the bench-size model: 64 x 2048-ray synthetic scans, 16 keyframes (p_th above 1 promotes every scan, so 20 scans fill the
model and evict).  Each build tree (this one, and optionally others given with --tree, e.g. a checkout of an earlier
commit built in place) runs in a process of its own, the trees alternating, --rounds times; a tree without the array
calls times the lists only.  Prints the card and its power limit with one JSON line per process.

    python scripts/leaves_bench.py [--tree /path/to/other/checkout] [--rounds 3] [--calls 50] [--out results.jsonl]
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def worker(root, scans_path, calls):
    sys.path.insert(0, root)
    import numpy as np
    import torch
    from mad_icp_b200.pybind.pypeline import Pipeline
    scans = list(np.load(scans_path).values())
    p = Pipeline(sensor_hz=10.0, deskew=False, b_max=0.2, rho_ker=0.1, p_th=1.5, b_min=0.1, b_ratio=0.02, num_keyframes=16,
                 num_threads=8, realtime=False)
    for i, c in enumerate(scans):
        p.compute(0.1 * i, c)
    assert p.numKeyframes() == 16
    stream = torch.cuda.current_stream()
    arms = {"currentLeaves": lambda: p.currentLeaves(), "modelLeaves": lambda: p.modelLeaves()}
    if hasattr(p, "modelLeavesArray"):
        arms.update({"currentLeavesArray": lambda: p.currentLeavesArray(),
                     "modelLeavesArray": lambda: p.modelLeavesArray(),
                     "currentLeavesArray(device=True)": lambda: (p.currentLeavesArray(device=True), stream.synchronize()),
                     "modelLeavesArray(device=True)": lambda: (p.modelLeavesArray(device=True), stream.synchronize())})
    ref = {"current": np.asarray(p.currentLeaves()), "model": np.asarray(p.modelLeaves())}
    ms = {}
    for name, fn in arms.items():
        for _ in range(3):  # warm-up: first allocations of the staging buffers
            fn()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(calls):
            fn()
        ms[name] = round((time.perf_counter() - t0) * 1e3 / calls, 4)
    same = True
    if hasattr(p, "modelLeavesArray"):
        same = (p.currentLeavesArray().tobytes() == ref["current"].tobytes() and
                p.modelLeavesArray(device=True).cpu().numpy().tobytes() == ref["model"].tobytes())
    return dict(leaves_current=int(ref["current"].shape[0]), leaves_model=int(ref["model"].shape[0]),
                digest_model=hashlib.sha256(ref["model"].tobytes()).hexdigest()[:16], arrays_equal_lists=bool(same), ms_per_call=ms)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [s.strip() for s in q.split(",")]
        return name, limit
    except Exception as e:  # (the table is still printed; the card is then "unknown")
        return f"unknown ({e})", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tree", action="append", default=[], help="another built checkout to time against this one")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", nargs=2, metavar=("ROOT", "SCANS"), help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        print(json.dumps(worker(a.worker[0], a.worker[1], a.calls)), flush=True)
        return
    import tempfile

    import numpy as np
    sys.path.insert(0, HERE)
    from mad_icp_b200 import synth
    name, limit = card()
    print(f"card: {name}, power limit {limit}", flush=True)
    trees = [os.path.abspath(t) for t in a.tree] + [HERE]
    lines = []
    with tempfile.TemporaryDirectory() as tmp:
        scans_path = os.path.join(tmp, "scans.npz")
        np.savez(scans_path, *synth.sequence(20, 64, 2048, workers=8)["scans"])
        for r in range(a.rounds):
            for t in trees:
                proc = subprocess.run([sys.executable, os.path.abspath(__file__), "--calls", str(a.calls), "--worker", t,
                                       scans_path], capture_output=True, text=True)
                if proc.returncode:
                    sys.exit(f"{t}: worker failed\n{proc.stderr}")
                out = proc.stdout
                row = dict(json.loads(out.strip().splitlines()[-1]), tree=t, round=r, card=name, power_limit=limit)
                print(json.dumps(row), flush=True)
                lines.append(row)
    if a.out:
        with open(a.out, "w") as f:
            for row in lines:
                f.write(json.dumps(row) + "\n")


if __name__ == "__main__":
    main()
