"""Per-round timeline of the persistent kernel on one clock (%globaltimer) + CTA 0's fold trace, and A/B of kernel
variants: `make -C mad_icp_b200/csrc probe DEFS=... TAG=name` builds scripts/_bin/libmadicp_<name>.so; this script
runs itself once per library found there (one process each) and once for the product library.
    python scripts/tail_probe.py"""
import glob, os, subprocess, sys
sys.path.insert(0, os.getcwd())
if len(sys.argv) < 2:
    libs = sorted(glob.glob(os.path.join(os.getcwd(), "scripts", "_bin", "libmadicp_*.so")))
    for lib in libs + ["product"]:
        subprocess.run([sys.executable, __file__, lib], check=False)
    sys.exit(0)
import numpy as np, torch
from mad_icp_b200 import _capi
if sys.argv[1] != "product":
    _capi.LIB_PATH = sys.argv[1]
from mad_icp_b200 import FlatTree, Registrar, synth
print(f"== {os.path.basename(_capi.LIB_PATH)}", flush=True)
case = synth.registration_case(K=16)
reg = Registrar(device=0, max_keyframes=16)
for s in range(16):
    reg.put_keyframe(s, FlatTree(case["scans"][s]), T=case["kf_poses"][s])
reg.set_moving(FlatTree(case["query"]).leaf_means())
st = torch.cuda.Stream(); reg.set_stream(st.cuda_stream)
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
X0 = case["T_guess"]
def timed(iters, cold, n=30):
    ts = []
    for _ in range(n):
        if cold:
            with torch.cuda.stream(st): flush.fill_(1)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(st); reg.register_async(X0, iters); b.record(st); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    return np.median(ts)
reg.set_gn_grid(768, 1)
reg.debug_timing(False, fetch=False)
out = reg.register(X0, 10)
walked = reg.register_walked() if hasattr(reg, "register_walked") else None
print(f"   n_matched {out['n_matched']}  pose_t {out['X'][:, 3].tolist()}  walked/round {walked if walked is None else list(walked)}")
print(f"   it1 {timed(1, False):.1f}  it5 {timed(5, False):.1f}  it10 warm {timed(10, False):.1f} cold {timed(10, True):.1f}  it15 {timed(15, False):.1f} us", flush=True)
reg.debug_timing(True, fetch=False)
for _ in range(3):
    reg.register_async(X0, 10); torch.cuda.synchronize()
d = reg.debug_timing(True)
start, end, pub = (reg.debug_cta_stamps(p, 10).astype(np.float64) for p in (1, 2, 3))
folded, handed = d[:, 6].astype(np.float64), d[:, 7].astype(np.float64)
ghz = torch.cuda.get_device_properties(0).clock_rate * 1e-6  # the device's SM clock (kHz -> GHz)
print("   CTA 0 (cycles): fold wait", d[:, 2].tolist(), " solve+publish", d[:, 4].tolist())
for it in (0, 3, 8):
    t0 = start[it].min()
    rel = lambda a: (a - t0) * ghz  # ns -> SM cycles (the timer ticks every ~256 ns)
    print(f"   round {it} (cycles after the first CTA started): items end min/p50/max {rel(end[it]).min():.0f}/{np.median(rel(end[it])):.0f}/{rel(end[it]).max():.0f}"
          f"  tile out max {rel(pub[it]).max():.0f}  folded {rel(folded[it]):.0f}  pose out {rel(handed[it]):.0f}"
          f"  next starts min/p50/max {rel(start[it + 1]).min():.0f}/{np.median(rel(start[it + 1])):.0f}/{rel(start[it + 1]).max():.0f}")
tr = reg.debug_cta_stamps(4, 10)[:, :16]
for it in (3, 8):
    t = tr[it]
    sweeps = int(t[14])
    marks = [int(x - t[0]) for x in t[1:1 + min(sweeps, 12)]]
    print(f"   round {it} fold trace (cycles after CTA 0 entered the fold): thread 0's sweeps end at {marks} ({sweeps} sweeps), fold done {int(t[13] - t[0])}")
reg.debug_timing(False, fetch=False)
reg.set_gn_grid(0, 1)
print(f"   auto shape: 10 iters warm/cold {timed(10, False):.1f} / {timed(10, True):.1f}", flush=True)
