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
    # the reference's -DUSE_HDF5=yes build: the default library plus the -st=h5 file writer
    "hdf5": ("libdenseflow_b200_hdf5.so", ["-DDFB_USE_HDF5=1"]),
    # the strict library with the writer: lets tests compare the command's h5 files with the oracle
    "strict_hdf5": ("libdenseflow_b200_strict_hdf5.so", ["-DDFB_STRICT_FP", "-fmad=false", "-prec-div=true", "-prec-sqrt=true",
                                                         "-DDFB_USE_HDF5=1"]),
}

# Variants whose macro only some translation units read: (the variant whose objects they link for every other source, those
# sources).  Only the listed sources are compiled again.
RELINKED = {"hdf5": ("default", ("h5_writer.cu",)), "strict_hdf5": ("strict", ("h5_writer.cu",))}

DEFAULT_VARIANTS = ("default", "strict", "hdf5", "strict_hdf5")


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


def build(variants=DEFAULT_VARIANTS, verbose=False, force=False):
    os.makedirs(LIBDIR, exist_ok=True)
    hm = _headers_mtime()
    outs = []
    # a relinked variant's base is built first (its objects must be current)
    order = []
    for v in variants:
        if v in RELINKED and RELINKED[v][0] not in order:
            order.append(RELINKED[v][0])
        if v not in order:
            order.append(v)
    for v in order:
        out_name, extra = VARIANTS[v]
        base, own = RELINKED.get(v, (v, None))
        objdir = os.path.join(LIBDIR, "obj_" + v)
        os.makedirs(objdir, exist_ok=True)
        jobs = []
        objs = []
        for src in _sources():
            sp = os.path.join(CSRC, src)
            if own is not None and src not in own:
                objs.append(os.path.join(LIBDIR, "obj_" + base, src[:-3] + ".o"))
                continue
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
        if jobs or not os.path.exists(out) or any(os.path.getmtime(o) > os.path.getmtime(out) for o in objs):
            _run([NVCC] + ARCH + ["-shared", "-o", out] + objs + ["-cudart", "shared", "-ldl", "-Xlinker", "-rpath=/usr/local/cuda/lib64"])
        if v in variants:
            outs.append(out)
    return outs


if __name__ == "__main__":
    names = tuple(a for a in sys.argv[1:] if a in VARIANTS) or DEFAULT_VARIANTS
    print("\n".join(build(names, verbose="-v" in sys.argv, force="-f" in sys.argv)))
