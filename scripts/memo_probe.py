"""Persistent-kernel timing in the three path-memo modes; per-round walk counts, quad records loaded and phase stamps.
python scripts/memo_probe.py [threads,ctas ...]"""
import os, sys
sys.path.insert(0, os.getcwd())
import numpy as np, torch
from mad_icp_b200 import FlatTree, Registrar, synth
case = synth.registration_case(K=16)
reg = Registrar(device=0, max_keyframes=16)
for s in range(16):
    reg.put_keyframe(s, FlatTree(case["scans"][s]), T=case["kf_poses"][s])
reg.set_moving(FlatTree(case["query"]).leaf_means())
st = torch.cuda.Stream(); reg.set_stream(st.cuda_stream)
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
X0 = case["T_guess"]
def timed(iters, cold, n=20):
    ts = []
    for _ in range(n):
        if cold:
            with torch.cuda.stream(st): flush.fill_(1)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(st); reg.register_async(X0, iters); b.record(st); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    return np.median(ts)
for shape in tuple(tuple(int(v) for v in a.split(',')) for a in sys.argv[1:]) or ((768, 1), (704, 1), (1024, 1)):
    reg.set_gn_grid(*shape)
    for memo in (2, 1, 0):  # leaf memo + resume, leaf memo only, every pair walked from the root
        reg.set_memo(memo)
        reg.debug_timing(False, fetch=False)
        line = f"shape {shape} memo={memo}:"
        for iters in (1, 2, 5, 10, 15):
            line += f"  it{iters}: {timed(iters, False):.1f}/{timed(iters, True):.1f}"
        print(line + "  us warm/cold", flush=True)
        reg.debug_timing(True, fetch=False)
        for _ in range(2):
            reg.register_async(X0, 10); torch.cuda.synchronize()
        d = reg.debug_timing(True)
        print("   per round: walked items (CTA 0)", d[:, 5].tolist())
        print("   per round: walked items (all)", reg.register_walked().tolist(), "quad records loaded",
              reg.register_walk_records().tolist())
        print("   per round: warp0/CTA0 items", d[:, 0].tolist(), "all folded", d[:, 1].tolist(), "fold wait", d[:, 2].tolist(), "solve", d[:, 4].tolist())
        cta = reg.debug_cta_cycles(10)
        print("   per-CTA item phase: round 0 min/p50/max", int(cta[0].min()), int(np.median(cta[0])), int(cta[0].max()),
              " round 9:", int(cta[9].min()), int(np.median(cta[9])), int(cta[9].max()), "slowest", np.argsort(cta[9])[-4:].tolist())
reg.set_gn_grid(0, 1); reg.set_memo(True)
reg.debug_timing(False, fetch=False)
print("auto shape, memo on: 10 iters warm/cold", timed(10, False), timed(10, True))
