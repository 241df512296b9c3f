"""In-tree build of the CUDA extension: nvcc -> denseflow_b200/lib/libdenseflow_b200.so (sm_90a only).

Called by __graft_entry__.build(). nvcc cross-compiles without a GPU. The .so is a build product and
is git-ignored.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC,-Wall,-Wno-unused-function", "-ccbin", "g++",
          "-I", os.path.join(HERE, "..", "include")]

VARIANTS = {
    # name: (output, extra flags)
    "default": ("libdenseflow_b200.so", []),
    # IEEE arithmetic, no FMA contraction: used by tests to separate restatement bugs from fp noise
    "strict": ("libdenseflow_b200_strict.so", ["-DDFB_STRICT_FP", "-fmad=false", "-prec-div=true", "-prec-sqrt=true"]),
    # geometry experiments of the fused tvl1 kernel (not built by default): python -m denseflow_b200.build t256
    "t256": ("libdenseflow_b200_t256.so", ["-DDFB_FUSED_THREADS=256"]),
    "t512": ("libdenseflow_b200_t512.so", ["-DDFB_FUSED_THREADS=512"]),
    "fb4": ("libdenseflow_b200_fb4.so", ["-DDFB_FARN_TMA_MINB=4"]),  # Farneback TMA kernel at 4 CTAs / SM (64 registers)
    "fb3": ("libdenseflow_b200_fb3.so", ["-DDFB_FARN_TMA_MINB=3"]),
    # arithmetic experiments of the TV-L1 inner loop (default build only differs by these flags)
    "mB": ("libdenseflow_b200_mB.so", ["-DDFB_TWO_RCP"]),  # two reciprocals per pixel in the dual step instead of the shared one
    "hx6": ("libdenseflow_b200_hx6.so", ["-DDFB_FARN_HX=6"]),  # Farneback window without the 32-byte origin alignment
}


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _headers_mtime():
    hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hs.append(os.path.join(HERE, "..", "include", "denseflow_b200.h"))
    return max(os.path.getmtime(h) for h in hs)


def _run(cmd):
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("command failed: %s\n%s\n%s" % (" ".join(cmd), r.stdout, r.stderr))
    return r.stdout + r.stderr


def build(variants=("default", "strict"), verbose=False, force=False):
    os.makedirs(LIBDIR, exist_ok=True)
    hm = _headers_mtime()
    outs = []
    for v in variants:
        out_name, extra = VARIANTS[v]
        objdir = os.path.join(LIBDIR, "obj_" + v)
        os.makedirs(objdir, exist_ok=True)
        jobs = []
        objs = []
        for src in _sources():
            sp = os.path.join(CSRC, src)
            obj = os.path.join(objdir, src[:-3] + ".o")
            objs.append(obj)
            if force or not os.path.exists(obj) or os.path.getmtime(obj) < max(os.path.getmtime(sp), hm):
                cmd = [NVCC] + ARCH + COMMON + extra + ["-c", sp, "-o", obj]
                if verbose:
                    cmd.insert(1, "-Xptxas=-v")
                jobs.append(cmd)
        with ThreadPoolExecutor(max_workers=8) as ex:
            for log in ex.map(_run, jobs):
                if verbose and log.strip():
                    print(log)
        out = os.path.join(LIBDIR, out_name)
        if jobs or not os.path.exists(out):
            _run([NVCC] + ARCH + ["-shared", "-o", out] + objs + ["-cudart", "shared", "-ldl", "-Xlinker", "-rpath=/usr/local/cuda/lib64"])
        outs.append(out)
    return outs


if __name__ == "__main__":
    names = tuple(a for a in sys.argv[1:] if a in VARIANTS) or ("default", "strict")
    print("\n".join(build(names, verbose="-v" in sys.argv, force="-f" in sys.argv)))
