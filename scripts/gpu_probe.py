"""GPU timing probe (not a bench line): warm/cold cost of the search kernel and of the persistent
GN kernel as a function of the round count.  Usage: python scripts/gpu_probe.py [K] """
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from mad_icp_b200 import FlatTree, Registrar, synth

K = int(sys.argv[1]) if len(sys.argv) > 1 else 16
case = synth.registration_case(K=K)
reg = Registrar(device=0, max_keyframes=K)
st = torch.cuda.Stream()
reg.set_stream(st.cuda_stream)
for s in range(K):
    ft = FlatTree(case["scans"][s]); ft.apply_transform(case["kf_poses"][s]); reg.put_keyframe(s, ft)
means = FlatTree(case["query"]).leaf_means()
reg.set_moving(torch.from_numpy(means).pin_memory())
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
X0 = case["T_guess"]

def timed(fn, n=30, cold=False):
    ts = []
    for _ in range(n):
        if cold:
            with torch.cuda.stream(st): flush.fill_(1)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(st); fn(); b.record(st); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    ts.sort()
    return ts[len(ts) // 2], ts[0]

print(f"K={K} L={means.shape[0]} items/round={K*means.shape[0]}")
for iters in (1, 2, 5, 10, 15, 20):
    w = timed(lambda: reg.register_async(X0, iters))
    c = timed(lambda: reg.register_async(X0, iters), cold=True)
    print(f"gn_loop iters={iters:2d}: warm median {w[0]:8.1f} us (min {w[1]:8.1f})   cold median {c[0]:8.1f} us (min {c[1]:8.1f})")

# per-round phase breakdown (SM cycles) per walk mode and shape
reg.debug_timing(True, fetch=False)
for mode in (4, 1):
    pass
    for thr, cps in ((1024, 1), (768, 1)):
        reg.set_gn_grid(thr, cps)
        w = timed(lambda: reg.register_async(X0, 10))
        reg.register_async(X0, 10); torch.cuda.synchronize()
        d = reg.debug_timing(True)
        cta = reg.debug_cta_cycles(10)[1:]          # skip the cold first round
        med = np.median(cta, axis=0)                # per-CTA median over rounds
        order = np.argsort(med)
        rho = np.corrcoef(cta[0], cta[-1])[0, 1]    # are the same CTAs slow in every round?
        print(f"mode={mode} shape=({thr},{cps}): 10-iter warm {w[0]:.1f} us | round cycles: all_arrived={np.median(d[:,1]):.0f} "
              f"fold={np.median(d[:,2]):.0f} solve={np.median(d[:,4]):.0f} | per-CTA item phase: min={med.min():.0f} "
              f"p50={np.median(med):.0f} p90={np.percentile(med,90):.0f} max={med.max():.0f} slowest CTAs={order[-4:].tolist()} "
              f"fastest={order[:4].tolist()} round-to-round corr={rho:.2f}")
pass
