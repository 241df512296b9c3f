"""Static instruction mix of the fused TV-L1 tile loop (runs without a GPU).

  python scripts/sass_loop_mix.py [variant]        variant of denseflow_b200/build.py (default: "default")

Compiles tvl1_fused.cu for sm_90a with the flags of that build variant plus -lineinfo, prints what ptxas reports for
k_tvl1_pair<FusedBatchParams, false> (the kernel of launches with <= 16 lanes and no median filtering), and counts the SASS of one tile iteration of an
interior tile (tile_iterations<false>): the lean instantiation tile_iteration<false, false>, which runs all but the last
iteration of a checking chunk, and the ERR instantiation tile_iteration<false, true>.  An instruction belongs to an
instantiation when its inlining chain (nvdisasm -gi) passes through that call of tile_iteration inside the
tile_iterations<false> call of process_tile; the call sites are found in the source, so the script follows edits.
"""
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from denseflow_b200 import build as B  # noqa: E402

SRC = os.path.join(B.CSRC, "tvl1_fused.cu")
KERNEL = "k_tvl1_pairINS_16FusedBatchParamsELb0E"
CUDA_BIN = os.path.dirname(B.NVCC)


def call_lines():
    """Source lines of the three calls that identify the interior-tile instantiations."""
    want = {"lean": "tile_iteration<EDGE, false>(", "err": "tile_iteration<EDGE, true>(", "interior": "tile_iterations<false>("}
    found = {}
    with open(SRC) as f:
        for i, line in enumerate(f, 1):
            for k, s in want.items():
                if s in line:
                    found[k] = i
    missing = set(want) - set(found)
    if missing:
        raise SystemExit("call sites not found in %s: %s" % (SRC, sorted(missing)))
    return found


def compile_cubin(variant, out):
    extra = B.VARIANTS[variant][1]
    cmd = [B.NVCC] + B.ARCH + B.COMMON + extra + ["-Xptxas", "-v", "-cubin", SRC, "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True, check=True)
    log = (r.stdout + r.stderr).splitlines()
    lines = []
    for i, l in enumerate(log):
        if "Compiling entry function" in l and KERNEL in l:
            lines = [x.split(":", 1)[-1].strip() for x in log[i + 1:i + 4] if "Function properties" not in x]
    return lines


def parse_sass(cubin):
    """[(opcode, chain)] for the pair kernel, chain = the (file, line) pairs of its inlining chain"""
    txt = subprocess.run([os.path.join(CUDA_BIN, "nvdisasm"), "-c", "-gi", cubin], capture_output=True, text=True, check=True).stdout
    loc = re.compile(r'File "([^"]+)", line (\d+)(?: inlined at "([^"]+)", line (\d+))?')
    ins = re.compile(r'^\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P[T0-9]\s+)?([A-Z0-9_]+)(\.[A-Z0-9_.]+)?')
    label = re.compile(r'^(\.L_x_\d+):')
    target = re.compile(r'`\((\.L_x_\d+)\)')
    out, labels, inside = [], {}, False
    lines, fresh = set(), True  # fused.cu lines of the current location's chain; fresh: the next "//## File" starts a new chain
    for line in txt.splitlines():
        if line.startswith(".text."):
            inside = KERNEL in line
            continue
        if not inside:
            continue
        m = label.match(line)
        if m:
            labels[m.group(1)] = len(out)
            continue
        m = loc.search(line)
        if m and "//##" in line:
            if fresh:
                lines, fresh = set(), False
            for f, n in ((m.group(1), m.group(2)), (m.group(3), m.group(4))):
                if f and os.path.basename(f) == "tvl1_fused.cu":
                    lines.add(int(n))
            continue
        m = ins.match(line)
        if m:
            t = target.search(line) if m.group(1) == "BRA" else None
            out.append((m.group(1), m.group(1) + (m.group(2) or ""), lines, t.group(1) if t else None))
            fresh = True
    return [(op, full, ls, labels.get(t)) for op, full, ls, t in out]


def owned(instr, call, interior):
    return call in instr[2] and interior in instr[2]


def loops(instrs, call, interior):
    """Bodies [head, branch] of the loops (backward branches) whose instructions are nearly all the given instantiation:
    the iteration loop of tile_iterations, once per copy ptxas made of it (spin loops of the flag waits excluded)"""
    found = []
    for i, (op, full, ls, tgt) in enumerate(instrs):
        if op == "BRA" and tgt is not None and tgt < i:
            body = instrs[tgt:i + 1]
            if len(body) > 64 and sum(owned(x, call, interior) for x in body) >= 0.9 * len(body):
                found.append(body)
    return found


def mix(instrs):
    return collections.Counter(x[0] for x in instrs), collections.Counter(x[1] for x in instrs)


def report(name, ops, full):
    total = sum(ops.values())
    print("  %-36s %4d instructions = %.1f per pixel-iteration (16 px per thread)" % (name, total, total / 16.0))
    fp32 = ops["FFMA"] + ops["FADD"] + ops["FMUL"]
    print("    FP32 %d (FFMA %d, FADD %d, FMUL %d), FMNMX %d, MUFU %d | MOV %d (+ IMAD.MOV %d), LDS %d, STS %d, SHFL %d, "
          "LDL %d, STL %d, S2R %d, MEMBAR %d" % (fp32, ops["FFMA"], ops["FADD"], ops["FMUL"], ops["FMNMX"], ops["MUFU"], ops["MOV"],
                                                 full["IMAD.MOV.U32"] + full["IMAD.MOV"], ops["LDS"], ops["STS"], ops["SHFL"],
                                                 ops["LDL"], ops["STL"], ops["S2R"], ops["MEMBAR"]))
    print("    all: " + ", ".join("%s %d" % kv for kv in sorted(ops.items(), key=lambda kv: (-kv[1], kv[0]))))


def main():
    variant = sys.argv[1] if len(sys.argv) > 1 else "default"
    cl = call_lines()
    with tempfile.TemporaryDirectory() as td:
        cubin = os.path.join(td, "tvl1_fused.cubin")
        ptxas = compile_cubin(variant, cubin)
        instrs = parse_sass(cubin)
    print("build variant %r, k_tvl1_pair<FusedBatchParams, false>, sm_90a" % variant)
    for l in ptxas:
        print("  ptxas: " + l)
    for n, body in enumerate(loops(instrs, cl["lean"], cl["interior"])):
        report("lean loop body, copy %d" % n, *mix(body))
    report("ERR iteration (all its code)", *mix([x for x in instrs if owned(x, cl["err"], cl["interior"])]))


if __name__ == "__main__":
    main()
