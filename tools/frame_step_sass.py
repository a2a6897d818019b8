"""Static cost of one frame step of the fused TSDF update, read from the compiled SASS (no GPU needed).
Compiles b2v_tsdf.cu with build.py's flags for sm_90a, finds the frame loop of `integrate_group_kernel` and prints,
as one JSON line:
    hot_per_frame   instructions on the hot path of one frame step, by opcode class: the frame loop from its head to
                    its back edge, halved because the loop is unrolled by two.  Left out: the blocks that only the
                    exact-division fallbacks reach (the `rare` projection path and the div_rn_slow calls of the
                    update), and the body of the z-step loop, which runs 0..3 times per frame and is given apart
    z_step          instructions per iteration of the z-step loop, per frame step
    kernels         registers and spill bytes of integrate_group_kernel and integrate_kernel (ptxas -v)
    checks          no spills in either kernel, and no 64-bit address arithmetic per gather on the hot path; the
                    exit status is 1 when a check fails
Cold code is found by its calls (div_rn_slow is the only callee of the update kernels): the outermost reconvergence
region (BSSY .. BSYNC) around a call is cold past the branch that skips it, and a call outside such a region is cold
from the forward branch that steps over it to that branch's target.
python tools/frame_step_sass.py [--rev GIT_REV]   (--rev: the sources of another commit, e.g. HEAD~1)"""
import argparse
import collections
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pyslam_b200 import build as B  # noqa: E402

GROUP = "integrate_group_kernel"
KERNELS = (GROUP, "integrate_kernel")
CLASSES = [  # first match wins; an opcode no class names is counted as "other"
    ("control", r"(BRA|BRX|JMP|JMX|CALL|RET|EXIT|BSSY|BSYNC|BREAK|WARPSYNC|BAR|NOP|YIELD)$"),
    ("vote", r"(VOTE|VOTEU|MATCH|SHFL|REDUX)$"),
    ("memory", r"(LDG|STG|LDS|STS|LDC|ULDC|LD|ST|ATOM|ATOMG|ATOMS|RED|LDL|STL)$"),
    ("move", r"(MOV|UMOV|S2R|S2UR|CS2R|R2UR|MOV32I)$|HFMA2\.MMA|IMAD\.MOV"),
    ("select/predicate", r"(SEL|FSEL|USEL|PLOP3|UPLOP3|P2R|R2P)$"),
    ("fp32", r"(FADD|FMUL|FFMA|FMNMX|FSETP|FSET|MUFU|FCHK|FSWZADD)$"),
    ("int/logic", r"(IADD3|IMAD|LOP3|SHF|ISETP|LEA|PRMT|FLO|POPC|BREV|I2F|F2I|F2F|IABS|IMNMX|"
                  r"UIADD3|UIMAD|ULOP3|USHF|UISETP|ULEA|UPRMT|UFLO|UPOPC|UBREV)$"),
]


def classify(op):
    for name, pat in CLASSES:
        if re.match(pat, op) or re.match(pat, op.split(".")[0]):
            return name
    return "other"


def sources(rev, dst):
    if rev is None:
        return os.path.join(ROOT, "pyslam_b200", "csrc")
    tar = subprocess.run(["git", "-C", ROOT, "archive", rev, "pyslam_b200/csrc", "include"], check=True,
                         capture_output=True).stdout
    subprocess.run(["tar", "-x", "-C", dst], input=tar, check=True)
    return os.path.join(dst, "pyslam_b200", "csrc")


def compile_tsdf(csrc, tmp):
    obj = os.path.join(tmp, "b2v_tsdf.o")
    nvcc = B._nvcc()
    r = subprocess.run([nvcc, *B.NVCC_FLAGS, "-Xptxas", "-v", "-c", os.path.join(csrc, "b2v_tsdf.cu"), "-o", obj],
                       capture_output=True, text=True)
    if r.returncode:
        raise SystemExit(r.stdout + r.stderr)
    kernels, cur = {}, None
    for line in (r.stdout + r.stderr).splitlines():
        # every function ptxas reports on (kernels and the noinline callees) opens with one of these two lines
        m = re.search(r"(?:Compiling entry function '|Function properties for )(\S+?)'?$", line)
        if m:
            cur = next((k for k in KERNELS if f"{len(k)}{k}E" in m.group(1)), None)
            continue
        if cur and "spill stores" in line:
            s = re.findall(r"(\d+) bytes spill (stores|loads)", line)
            kernels.setdefault(cur, {}).update({f"spill_{kind}": int(n) for n, kind in s})
        if cur and "Used" in line and "registers" in line:
            kernels.setdefault(cur, {})["registers"] = int(re.search(r"Used (\d+) registers", line).group(1))
    cuobj = shutil.which("cuobjdump") or os.path.join(os.path.dirname(nvcc), "cuobjdump")
    sass = subprocess.run([cuobj, "-sass", obj], check=True, capture_output=True, text=True).stdout
    return kernels, sass


def function_sass(sass, kernel):
    """[(address, predicate, opcode, operands)] of the kernel's function."""
    out, on = [], False
    for line in sass.splitlines():
        if "Function :" in line:
            on = f"{len(kernel)}{kernel}E" in line
            continue
        if not on:
            continue
        m = re.match(r"\s*/\*([0-9a-f]+)\*/\s+(@!?U?P[T0-9]+\s+)?([A-Z0-9_.]+)\s*(.*?)\s*;", line)
        if m:
            out.append((int(m.group(1), 16), (m.group(2) or "").strip(), m.group(3), m.group(4)))
    return out


def blocks_of(ins):
    addr = {a: i for i, (a, *_) in enumerate(ins)}
    target = {}
    leaders = {0}
    for i, (a, pred, op, args) in enumerate(ins):
        if op.startswith(("BRA", "EXIT", "RET", "BRX", "JMP")):
            m = re.findall(r"0x([0-9a-f]+)", args)
            if op.startswith("BRA") and m:
                target[i] = addr[int(m[-1], 16)]
                leaders.add(target[i])
            leaders.add(i + 1)
    starts = sorted(s for s in leaders if s < len(ins))
    blk = {}
    for bi, s in enumerate(starts):
        e = starts[bi + 1] if bi + 1 < len(starts) else len(ins)
        blk[s] = list(range(s, e))
    succ = {}
    for s, body in blk.items():
        last = body[-1]
        pred, op = ins[last][1], ins[last][2]
        nxt = [last + 1] if last + 1 < len(ins) else []
        conditional = pred not in ("", "@PT")
        if op.startswith("BRA"):
            succ[s] = [target[last]] + (nxt if conditional else [])
        elif op.startswith(("EXIT", "RET")):
            succ[s] = nxt if conditional else []
        else:
            succ[s] = nxt
    return blk, succ


def dominators(nodes, succ, entry):
    preds = {n: [p for p in nodes if n in succ[p]] for n in nodes}
    dom = {n: set(nodes) for n in nodes}
    dom[entry] = {entry}
    changed = True
    while changed:
        changed = False
        for n in nodes:
            if n == entry:
                continue
            ps = [dom[p] for p in preds[n]]
            d = set.intersection(*ps) | {n} if ps else {n}
            if d != dom[n]:
                dom[n], changed = d, True
    return dom


def natural_loop(head, latch, preds):
    body, stack = {head, latch}, [latch] if latch != head else []
    while stack:
        for p in preds[stack.pop()]:
            if p not in body:
                body.add(p)
                stack.append(p)
    return body


def analyse(ins):
    blk, succ = blocks_of(ins)
    nodes = sorted(blk)
    dom = dominators(nodes, succ, nodes[0])
    preds = {n: [p for p in nodes if n in succ[p]] for n in nodes}
    loops = [(h, u, natural_loop(h, u, preds)) for u in nodes for h in succ[u] if h in dom[u]]
    has = lambda b, pat: any(re.match(pat, ins[i][2]) for i in blk[b])  # noqa: E731
    # the frame loop: the largest loop without a CTA barrier (the work loop around it has one per block)
    head, latch, body = max((lp for lp in loops if not any(has(b, r"BAR") for b in lp[2])), key=lambda lp: len(lp[2]))
    inside = sorted(body)
    # cold: the outermost reconvergence regions (BSSY .. its BSYNC) that contain a call, except the instructions up to
    # the branch that skips the region and the BSYNC; a call outside such a region is cold from the forward branch
    # that skips it to that branch's target
    at = {a: i for i, (a, *_) in enumerate(ins)}
    regions = []
    for i, (a, pred, op, args) in enumerate(ins):
        if op.startswith("BSSY"):
            end = at[int(re.findall(r"0x([0-9a-f]+)", args)[-1], 16)]
            if any(ins[j][2].startswith("CALL") for j in range(i, end)):
                regions.append((i, end))
    regions = [r for r in regions if not any(o[0] < r[0] and r[1] <= o[1] for o in regions)]
    cold = set()
    for i, end in regions:
        j = i
        while j < end and not (ins[j][2].startswith("BRA") and ins[j][1] and
                               at[int(re.findall(r"0x([0-9a-f]+)", ins[j][3])[-1], 16)] >= end - 1):
            j += 1
        cold |= set(range(j + 1, end))
    for c, (a, pred, op, args) in enumerate(ins):
        if op.startswith("CALL") and c not in cold:
            g = max((j for j in range(c) if ins[j][2].startswith("BRA") and ins[j][1] and
                     at[int(re.findall(r"0x([0-9a-f]+)", ins[j][3])[-1], 16)] > c), default=None)
            if g is None:  # an unguarded call stays on the hot path
                continue
            cold |= set(range(g + 1, at[int(re.findall(r"0x([0-9a-f]+)", ins[g][3])[-1], 16)]))
    # a forward branch that skips nothing but cold code and control flow guards a cold region too (a warp-uniform
    # guard needs no BSSY)
    control = re.compile(r"(BSSY|BSYNC|BRA)")
    grown = True
    while grown:
        grown = False
        for g, (a, pred, op, args) in enumerate(ins):
            if op.startswith("BRA") and pred:
                tgt = at[int(re.findall(r"0x([0-9a-f]+)", args)[-1], 16)]
                span = range(g + 1, tgt)
                if tgt > g + 1 and not set(span) <= cold and any(j in cold for j in span) and \
                        all(j in cold or control.match(ins[j][2]) for j in span):
                    cold |= set(span)
                    grown = True
    # inner loops that stay hot (the z-step loop): counted per iteration, not in the frame step
    inner = [lp for lp in loops if lp[0] != head and lp[2] <= body and not any(set(blk[b]) & cold for b in lp[2])]
    zbody = set().union(*[lp[2] for lp in inner]) if inner else set()
    hot = [i for b in inside if b not in zbody for i in blk[b] if i not in cold]
    count = collections.Counter(classify(ins[i][2]) for i in hot)
    zcount = sum(len(blk[b]) for b in zbody) / 2
    return {
        "hot_per_frame": round(len(hot) / 2, 1),
        "by_class_per_frame": {k: round(v / 2, 1) for k, v in sorted(count.items())},
        "z_step": zcount,
        "loop_instructions": sum(len(blk[b]) for b in inside),
        "cold_instructions": sum(1 for b in inside for i in blk[b] if i in cold),
        "loop_span": [hex(ins[head][0]), hex(ins[blk[latch][-1]][0])],
        "indexed_ldc_per_frame": round(sum(1 for i in hot if ins[i][2].startswith("LDC") and "[R" in ins[i][3]) / 2, 1),
        # each gather's address should be one IMAD.WIDE of the pixel index on a per-frame base: 64-bit carry
        # arithmetic (LEA.HI.X, IADD3.X, IMAD.WIDE.U32) on the hot path means the compiler folded the frame's offset
        # into every gather again
        "wide_address_ops_per_frame": round(sum(1 for i in hot if re.match(r"(LEA\.HI\.X|IADD3\.X|IMAD\.WIDE\.U32)",
                                                                           ins[i][2])) / 2, 1),
    }


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--rev", default=None, help="analyse the sources of this git revision instead of the tree")
    args = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        kernels, sass = compile_tsdf(sources(args.rev, tmp), tmp)
    res = {"rev": args.rev or "working tree", **analyse(function_sass(sass, GROUP)), "kernels": kernels}
    res["checks"] = {"no_spills": all(k.get("spill_stores", 1) == 0 and k.get("spill_loads", 1) == 0
                                      for k in kernels.values()) and len(kernels) == len(KERNELS),
                     "no_wide_gather_addresses": res["wide_address_ops_per_frame"] == 0}
    print(json.dumps(res))
    return 0 if all(res["checks"].values()) else 1


if __name__ == "__main__":
    sys.exit(main())
