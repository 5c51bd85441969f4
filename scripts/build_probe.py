"""Host MAD-tree build timing as a function of the thread count (run it on a host with
many physical cores).  Usage: python scripts/build_probe.py"""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from mad_icp_b200 import FlatTree, synth

pts = synth.registration_case(K=1)["scans"][0]
print(f"host cores={os.cpu_count()} points={pts.shape[0]}")
for thr in (1, 4, 8, 16, 32, 64):
    ts = []
    for _ in range(8):
        t = time.perf_counter()
        ft = FlatTree(pts, num_threads=thr)
        ts.append(time.perf_counter() - t)
    ts.sort()
    print(f"threads={thr:2d}: build median {1e3 * ts[len(ts) // 2]:.2f} ms  min {1e3 * ts[0]:.2f} ms  nodes={ft.num_nodes}")
os.environ["MADTREE_TIMING"] = "1"
FlatTree(pts, num_threads=16)
FlatTree(pts, num_threads=16)
ft = FlatTree(pts, num_threads=16)
T = synth.pose_xyyaw(1.0, 2.0, 0.1)
t = time.perf_counter(); ft.apply_transform(T); print(f"apply_transform (16 threads) {1e3 * (time.perf_counter() - t):.2f} ms")
