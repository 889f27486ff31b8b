"""Build libsmot.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

Usage: python -m siammot_b200.build   (also called by __graft_entry__.build()).
"""
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libsmot.so")
STAMP = OUT + ".flags"   # the compiler, its version and FLAGS that built OUT: a change to any of them forces a rebuild
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC",
         "-fmad=false",  # contraction only where the kernels say fmaf(): coordinate maths stays IEEE like the CPU reference
         "--expt-relaxed-constexpr", "-cudart", "shared"]


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def toolchain_stamp():
    try:
        version = subprocess.run([NVCC, "--version"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True).stdout
    except OSError as exc:
        version = "unavailable: %s" % exc
    return "\n".join([NVCC, version.strip(), " ".join(FLAGS)]) + "\n"


def needs_build():
    if not os.path.exists(OUT) or not os.path.exists(STAMP):
        return True
    with open(STAMP) as f:
        if f.read() != toolchain_stamp():
            return True
    t = os.path.getmtime(OUT)
    deps = sources() + glob.glob(os.path.join(CSRC, "*.cuh")) + [os.path.join(HERE, "..", "include", "smot.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return OUT
    objs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    procs = []
    for src in sources():
        obj = os.path.join(HERE, "build", os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s" % (src, out))
        if verbose:
            print(out)
    tmp = OUT + ".tmp"   # link beside the target, then rename: a reader (or a repository snapshot) never sees a half-written library
    cmd = [NVCC, "-shared", "-cudart", "shared", "-o", tmp] + objs
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n%s" % r.stdout)
    os.replace(tmp, OUT)
    with open(STAMP, "w") as f:
        f.write(toolchain_stamp())
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
