"""SASS census of the persistent kernel in the built library: python scripts/sass_census.py [threads=768]
(cuobjdump -sass of mad_icp_b200/lib/libmadicp_b200.so, the k_gn_loop<threads,1> entry; counts by class, proof of what the
kernel does and does not use: DMMA yes, wgmma/TMA no)."""
import collections, os, re, subprocess, sys
threads = int(sys.argv[1]) if len(sys.argv) > 1 else 768
lib = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "mad_icp_b200", "lib", "libmadicp_b200.so")
txt = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
name = f"k_gn_loopILi{threads}ELi1E"
blocks = re.split(r"\n\s*Function : ", txt)
body = next(b for b in blocks if b.startswith("_ZN6madicp") and name in b.split("\n", 1)[0])
ops = collections.Counter()
for line in body.splitlines():
    m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
    if m:
        ops[m.group(1)] += 1
def cls(pred):
    sel = {k: v for k, v in ops.items() if pred(k)}
    return sum(sel.values()), ", ".join(f"{k}:{v}" for k, v in sorted(sel.items(), key=lambda kv: -kv[1])[:8])
rows = [
    ("DMMA (FP64 tensor pipe, mma.sync.m8n8k4.f64)", lambda k: k.startswith("DMMA")),
    ("LDG.E.128.CONSTANT (128-bit non-coherent loads: quad records, exact records, moving leaves)", lambda k: k.startswith("LDG.E.128.CONSTANT")),
    ("other LDG", lambda k: k.startswith("LDG") and not k.startswith("LDG.E.128.CONSTANT")),
    ("STG / ST (global stores)", lambda k: k.startswith("STG") or k == "ST" or k.startswith("ST.E")),
    ("LDL / STL (local memory: spills, call frames)", lambda k: k.startswith("LDL") or k.startswith("STL")),
    ("LDS / STS (shared memory)", lambda k: k.startswith("LDS") or k.startswith("STS")),
    ("FP64 arithmetic (DADD/DMUL/DFMA/DSETP)", lambda k: re.match(r"D(ADD|MUL|FMA|SETP)", k) is not None),
    ("FP32 arithmetic (FFMA/FMUL/FADD/FSETP/FMNMX)", lambda k: re.match(r"F(FMA|MUL|ADD|SETP|MNMX)", k) is not None),
    ("XU pipe: conversions + MUFU (F2F, F2I, I2F, MUFU.*)", lambda k: re.match(r"(F2F|F2I|I2F|MUFU)", k) is not None),
    ("wgmma / TMA (HGMMA, UTMALDG, UBLKCP)", lambda k: re.match(r"(HGMMA|UTMA|UBLKCP)", k) is not None),
    ("barriers / fences (BAR, MEMBAR, ERRBAR, CCTL)", lambda k: re.match(r"(BAR|MEMBAR|ERRBAR|CCTL)", k) is not None),
    ("warp collectives (SHFL, VOTE, MATCH, REDUX)", lambda k: re.match(r"(SHFL|VOTE|MATCH|REDUX)", k) is not None),
    ("atomics (ATOM*, RED.*)", lambda k: re.match(r"(ATOM|RED\.)", k) is not None),
]
print(f"# SASS census of k_gn_loop<{threads},1> (sm_90a cubin inside mad_icp_b200/lib/libmadicp_b200.so, cuobjdump -sass; scripts/sass_census.py)")
print(f"# {sum(ops.values())} instructions.  north_star: \"no tensor cores -- memory/branch bound\": no wgmma/TMA tiles; the only")
print("# tensor-pipe use is the FP64 DMMA fold of the per-correspondence outer products (register economy, DESIGN.md 4.3).\n")
for label, pred in rows:
    n, detail = cls(pred)
    print(f"{n:5d}  {label}" + (f"   [{detail}]" if n else ""))
print("\ntop 25 mnemonics: " + ", ".join(f"{k}:{v}" for k, v in ops.most_common(25)))
