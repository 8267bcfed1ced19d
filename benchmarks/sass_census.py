"""Static instruction census of the HighwayLite sub-step loop (`hw::step`) inside `opd_highway_multi_kernel`.

Compiles csrc/opd.cu to a cubin with the library's own nvcc flags (rl_agents_b200/build.py), disassembles it with
inline line information and counts, per issue pipe, the instructions whose source position inside `hw::step` lies in
the sub-step loop -- including what helpers inlined there (not_zero, idm_front, asin_p, ...) compiled to.  The scan
path (exact x ties), the rank recount (first sub-step, and after an overtake) and the collision loop are reported apart from the common
path.  CPU only: needs nvcc and nvdisasm, no GPU.

    python benchmarks/sass_census.py [--ops]

Pipe classes (Hopper): ALU = compares, selects, min/max, logic, shifts, integer add / LEA, bit counts (half-rate);
FMA = FFMA/FADD/FMUL (FMA-heavy or FMA-lite); FMA-heavy = IMAD/IMUL (FMA-heavy only); MIO = shared / local / global
memory, shuffles, votes, matches, MUFU; branch = control flow.
"""
import argparse
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rl_agents_b200 import build  # noqa: E402

KERNEL = "_ZN2b224opd_highway_multi_kernelENS_7OpdArgsE"
HEADER = os.path.join(build.CSRC, "highway_lite.cuh")

PIPES = {
    "ALU": {"FSETP", "ISETP", "FSEL", "SEL", "LOP3", "FMNMX", "IMNMX", "VIMNMX", "PLOP3", "SHF", "PRMT", "LEA",
            "IADD3", "FLO", "BREV", "POPC", "MOV", "P2R", "R2P"},
    "FMA": {"FFMA", "FADD", "FMUL"},
    "FMA-heavy": {"IMAD", "IMUL"},
    "MIO": {"LDS", "STS", "LDL", "STL", "LDG", "STG", "LD", "ST", "SHFL", "VOTE", "MATCH", "MUFU", "BAR", "S2R",
            "CS2R", "ATOMS", "REDUX"},
    "branch": {"BRA", "BSSY", "BSYNC", "WARPSYNC", "EXIT", "CALL", "RET", "BREAK", "JMP"},
}


def pipe_of(op):
    for name, ops in PIPES.items():
        if op in ops:
            return name
    return "other"


def block_end(lines, start):
    """1-based line of the brace that closes the block opened on line `start`."""
    depth = 0
    for i in range(start - 1, len(lines)):
        for ch in lines[i]:
            if ch == "{":
                depth += 1
            elif ch == "}":
                depth -= 1
                if depth == 0:
                    return i + 1
    raise ValueError("unbalanced block at line %d" % start)


def regions():
    """(loop range, {name: [ranges]}) of the sub-step loop and of the parts kept apart from its common path."""
    lines = open(HEADER).read().splitlines()

    def starts(pattern):
        return [i + 1 for i, l in enumerate(lines) if re.search(pattern, l)]

    loop = starts(r"for \(int sub = 0; sub <= SUBSTEPS; \+\+sub\)")
    assert len(loop) == 1, loop
    lo, hi = loop[0], block_end(lines, loop[0])
    inside = lambda ls: [(s, block_end(lines, s)) for s in ls if lo < s < hi]  # noqa: E731
    apart = {"scan path": inside(starts(r"if \(scan\) \{")),
             "rank recount": inside(starts(r"if \(!fresh\) \{")),
             "collision loop": inside(starts(r"for \(int k = 1; k < V; \+\+k\)"))}
    return (lo, hi), apart


def disassemble(workdir):
    cubin = os.path.join(workdir, "opd.cubin")
    flags = [f for f in build.NVCC_FLAGS if f not in ("--shared", "-Xcompiler", "-fPIC")]
    subprocess.run([os.environ.get("NVCC", "nvcc")] + flags + ["-cubin", "-o", cubin, os.path.join(build.CSRC, "opd.cu")],
                   check=True)
    return subprocess.run(["nvdisasm", "-gi", "-c", cubin], check=True, stdout=subprocess.PIPE, text=True).stdout


FRAME = re.compile(r'//## File "([^"]+)", line (\d+)(?: inlined at "([^"]+)", line (\d+))?')
INSN = re.compile(r"/\*[0-9a-f]+\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_]*)")


def census(sass):
    """Yield (opcode, step line, inlined helper?) for every instruction of the kernel that `hw::step` emitted."""
    in_kernel, frames, fresh = False, [], True
    for raw in sass.splitlines():
        if raw.startswith("//---------------------"):
            in_kernel = (".text." + KERNEL + " ") in raw + " "
            continue
        if not in_kernel:
            continue
        m = FRAME.search(raw)
        if m:
            if fresh:
                frames, fresh = [], False
            frames.append(m.groups())
            continue
        m = INSN.search(raw)
        if not m:
            continue
        fresh = True
        # the frame of step() itself: a highway_lite.cuh line inlined into a caller in another file
        step = [i for i, f in enumerate(frames) if f[0].endswith("highway_lite.cuh") and f[2]
                and not f[2].endswith("highway_lite.cuh")]
        if step:
            yield m.group(1).split(".")[0], int(frames[step[0]][1]), step[0] > 0


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--ops", action="store_true", help="also list the common path's ALU opcodes")
    a = ap.parse_args()
    (lo, hi), apart = regions()
    with tempfile.TemporaryDirectory() as tmp:
        sass = disassemble(tmp)
    counts = collections.defaultdict(collections.Counter)
    alu_ops = collections.Counter()
    for op, line, inlined in census(sass):
        if not lo <= line <= hi:
            continue
        part = next((n for n, rs in apart.items() if any(s <= line <= e for s, e in rs)), None)
        if part is None:
            part = "common path, inlined helpers" if inlined else "common path, loop lines"
            if pipe_of(op) == "ALU":
                alu_ops[op] += 1
        counts[part][pipe_of(op)] += 1
    cols = ["ALU", "FMA", "FMA-heavy", "MIO", "branch", "other"]
    print("hw::step sub-step loop (highway_lite.cuh:%d-%d) in %s, static SASS instructions" % (lo, hi, KERNEL))
    print("%-32s" % "" + "".join("%10s" % c for c in cols) + "%10s" % "total")
    rows = ["common path, loop lines", "common path, inlined helpers", "scan path", "rank recount", "collision loop"]
    common = collections.Counter()
    for r in rows:
        c = counts.get(r, collections.Counter())
        if r.startswith("common"):
            common += c
        print("%-32s" % r + "".join("%10d" % c[k] for k in cols) + "%10d" % sum(c.values()))
        if r == "common path, inlined helpers":
            print("%-32s" % "common path, all" + "".join("%10d" % common[k] for k in cols)
                  + "%10d" % sum(common.values()))
    if a.ops:
        print("common path ALU opcodes: " + ", ".join("%s %d" % kv for kv in alu_ops.most_common()))


if __name__ == "__main__":
    main()
