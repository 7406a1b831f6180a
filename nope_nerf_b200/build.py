"""Builds the in-tree CUDA library  nope_nerf_b200/libnope_nerf_b200.so  for sm_90a (H100) with nvcc.
No torch dependency: the library is a plain C-ABI shared object (include/nope_nerf_b200.h)."""
import os, subprocess, sys, shutil

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libnope_nerf_b200.so")
SOURCES = ["nnb_api.cu", "nnb_simt.cu", "nnb_misc.cu", "nnb_tc.cu", "nnb_refstage.cu", "nnb_collective.cu", "nnb_options.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC",
              "--expt-relaxed-constexpr", "-DNNB_WITH_TC"]


def _nvcc():
    return shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "nope_nerf_b200.h"), __file__]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False, out=None, tag=""):
    """out/tag: build an instrumented variant (NNB_EXTRA_NVCC_FLAGS) beside the product library"""
    global LIB
    if out:
        LIB = os.path.abspath(out)
    if not force and not needs_build():
        return LIB
    srcs = [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    flags = list(NVCC_FLAGS) + os.environ.get("NNB_EXTRA_NVCC_FLAGS", "").split()
    if not os.path.exists(os.path.join(CSRC, "nnb_tc.cu")):
        flags.remove("-DNNB_WITH_TC")
    objs = []
    bdir = os.path.join(HERE, "build"); os.makedirs(bdir, exist_ok=True)
    procs = []
    for s in srcs:
        o = os.path.join(bdir, os.path.basename(s) + tag + ".o")
        objs.append(o)
        cmd = [_nvcc()] + flags + (["-Xptxas", "-v"] if verbose else []) + ["-c", s, "-o", o]
        procs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for cmd, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode:
            sys.stderr.write(out)
        if p.returncode:
            raise RuntimeError("nvcc failed: " + " ".join(cmd))
    cmd = [_nvcc(), "-shared", "-o", LIB] + objs + ["-cudart", "static"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode:
        sys.stderr.write(r.stdout)
        raise RuntimeError("link failed")
    return LIB


if __name__ == "__main__":
    out = sys.argv[sys.argv.index("--out") + 1] if "--out" in sys.argv else None
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv, out=out, tag=".dbg" if out else ""))
