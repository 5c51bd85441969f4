"""SASS census of the persistent kernel in the built library.

python scripts/sass_census.py [threads=768]
    cuobjdump -sass of mad_icp_b200/lib/libmadicp_b200.so, the k_gn_loop<threads,1> entry; counts by class, proof of what
    the kernel does and does not use: DMMA yes, wgmma/TMA no.
python scripts/sass_census.py --loop-spills [threads ...]
    local-memory instructions (LDL / STL) inside the item loop of k_gn_loop<threads,1>, per shape (default: every shape
    of the table in capi.cu).

The item loop is the innermost loop that holds every DMMA of the kernel: the shortest backward branch whose range covers
them all.  An LDL / STL in that range counts unless its basic block (no branch target and no branch between them) also
holds a CALL: those save and restore live registers around the out-of-line exact side test (side_exact, side_exact_m)
and the slow paths of sqrt and the reciprocal, which run only when the fast path cannot decide.  Every other local
access in the loop is a spill or a stack array that each item pays for."""
import collections, os, re, subprocess, sys

LIB = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "mad_icp_b200", "lib", "libmadicp_b200.so")
SHAPES = (1024, 896, 768, 704, 640, 512)  # the one-CTA-per-SM instantiations (capi.cu: gn_shapes)
_INSN = re.compile(r"\s*/\*([0-9a-f]{4,})\*/\s+(@!?U?P\w+\s+)?([A-Z0-9_.]+)([^;]*);")


def sass(lib=LIB, tool="cuobjdump"):
    return subprocess.run([tool, "-sass", lib], capture_output=True, text=True, check=True).stdout


def kernel_body(txt, threads, ctas=1):
    name = f"k_gn_loopILi{threads}ELi{ctas}E"
    blocks = re.split(r"\n\s*Function : ", txt)
    return next(b for b in blocks if b.startswith("_ZN6madicp") and name in b.split("\n", 1)[0])


def instructions(body):
    """[(address, opcode, operands)] in address order."""
    out = []
    for line in body.splitlines():
        m = _INSN.match(line)
        if m:
            out.append((int(m.group(1), 16), m.group(3), m.group(4)))
    return out


def _branch_targets(ins):
    out = []
    for a, op, args in ins:
        if op.startswith(("BRA", "BSSY", "BRX", "JMP")):
            m = re.search(r"0x([0-9a-f]+)\s*$", args.strip())
            if m:
                out.append((a, op, int(m.group(1), 16)))
    return out


def item_loop_range(ins):
    """(first, last) address of the item loop: the shortest backward branch around every DMMA."""
    dmma = [a for a, op, _ in ins if op.startswith("DMMA")]
    if not dmma:
        raise ValueError("no DMMA in the kernel: cannot find the item loop")
    backs = [(t, a) for a, op, t in _branch_targets(ins) if op.startswith("BRA") and t <= min(dmma) and a >= max(dmma)]
    if not backs:
        raise ValueError("no backward branch encloses the DMMA fold")
    return min(backs, key=lambda b: b[1] - b[0])


def item_loop_local_ops(body):
    """(counted, excused): the LDL / STL of the item loop, as (address, opcode) lists; excused = in a block with a CALL."""
    ins = instructions(body)
    lo, hi = item_loop_range(ins)
    targets = {t for _, _, t in _branch_targets(ins)}
    counted, excused, block, has_call = [], [], [], False

    def close():
        (excused if has_call else counted).extend(block)

    for a, op, _ in ins:
        if a < lo or a > hi:
            continue
        if a in targets:  # a label starts a new block
            close()
            block, has_call = [], False
        if op.startswith(("LDL", "STL")):
            block.append((a, op))
        if op.startswith("CALL"):
            has_call = True
        if op.startswith(("BRA", "BRX", "JMP", "EXIT", "RET")):  # ... and a branch ends one
            close()
            block, has_call = [], False
    close()
    return counted, excused


def census(threads):
    body = kernel_body(sass(), threads)
    ops = collections.Counter(op for _, op, _ in instructions(body))

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
    counted, excused = item_loop_local_ops(body)
    print(f"\nitem loop: {len(counted)} LDL/STL counted, {len(excused)} around calls")
    print("top 25 mnemonics: " + ", ".join(f"{k}:{v}" for k, v in ops.most_common(25)))


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "--loop-spills":
        txt = sass()
        for t in (tuple(int(v) for v in sys.argv[2:]) or SHAPES):
            counted, excused = item_loop_local_ops(kernel_body(txt, t))
            print(f"k_gn_loop<{t},1>: {len(counted)} LDL/STL in the item loop"
                  + (" (" + ", ".join(f"{op}@{a:#x}" for a, op in counted) + ")" if counted else "")
                  + f"; {len(excused)} around calls")
    else:
        census(int(sys.argv[1]) if len(sys.argv) > 1 else 768)
