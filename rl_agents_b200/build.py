"""Build libb2planner.so in-tree with nvcc for the H100 (sm_90a).  The library is
compiled ahead of time, so nothing is JIT-compiled or cached at run time."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(CSRC, "libb2planner.so")
STAMP = LIB + ".cmd"          # signature() of the build that made the library
SOURCES = ["common.cu", "vi.cu", "vi_p2p.cu", "opd.cu", "opd_wave.cu", "gbop.cu", "mcts.cu", "mcts_reroot.cu", "mcts_wave.cu",
           "olop.cu",
           "mdp_gape.cu", "brue.cu", "sparse_sampling.cu", "sparse_sampling_levels.cu",
           "mcts_dpw.cu", "platypoos.cu", "ttc_vi.cu", "finite_step.cu", "selftest.cu", "host_api.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    # parity: every fp op is a single IEEE operation (no FMA contraction), IEEE div/sqrt, no FTZ
    "-fmad=false", "-prec-div=true", "-prec-sqrt=true", "-ftz=false",
    "--shared", "-Xcompiler", "-fPIC",
]


def sources():
    return [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]


def command():
    return [os.environ.get("NVCC", "nvcc")] + NVCC_FLAGS + ["-o", LIB] + sources()


def signature():
    """What the library depends on besides file contents: compiler, flags and source list (no absolute paths, so
    that a moved tree is not rebuilt)."""
    return " ".join([os.environ.get("NVCC", "nvcc")] + NVCC_FLAGS + SOURCES)


def needs_build():
    """True when the library is missing, was built by another command (flags, architecture, sources) or is older
    than a source or the public header."""
    if not os.path.exists(LIB) or not os.path.exists(STAMP):
        return True
    with open(STAMP) as f:
        if f.read() != signature():
            return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh"))]
    deps.append(os.path.join(os.path.dirname(HERE), "include", "b2_planner.h"))
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    cmd = command()
    proc = subprocess.run(cmd + (["-Xptxas", "-v"] if verbose else []), stdout=subprocess.PIPE,
                          stderr=subprocess.STDOUT, text=True)
    if proc.returncode != 0:
        raise RuntimeError("nvcc failed:\n%s\n%s" % (" ".join(cmd), proc.stdout))
    with open(STAMP, "w") as f:
        f.write(signature())
    if verbose:
        print(proc.stdout)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
