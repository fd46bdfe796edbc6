"""Builds libgrl_b200.so (sm_90a only) in-tree with nvcc.  No torch headers are involved: the library is a
plain C-ABI shared object (include/grl_b200.h) that the Python surface loads with ctypes."""
import glob
import os
import shutil
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, "csrc")
LIB = os.path.join(PKG, "libgrl_b200.so")
NVCC_FLAGS = [
    "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-v",
    # the host copies of the closed forms (csrc/grl_hd.h) must evaluate each IEEE operation as written, on any host ISA
    "-Xcompiler", "-ffp-contract=off",
]


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


STAMP = os.path.join(PKG, "build", "defines.stamp")  # the GRL_NVCC_DEFINES the objects / library were compiled with


def _defines():
    return " ".join(os.environ.get("GRL_NVCC_DEFINES", "").split())


def _stamp():
    try:
        with open(STAMP) as f:
            return f.read().strip()
    except OSError:
        return ""  # no stamp: a production build (no defines)


def _stale():
    if not os.path.exists(LIB):
        return True
    if _stamp() != _defines():  # an A/B build left behind (or asked for): never mistake it for the production library
        return True
    t = os.path.getmtime(LIB)
    deps = sources() + glob.glob(os.path.join(CSRC, "*.h")) + glob.glob(os.path.join(CSRC, "*.cuh"))
    deps.append(os.path.join(os.path.dirname(PKG), "include", "grl_b200.h"))
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    """Compile every .cu under csrc/ into one shared library.  Returns the library path."""
    if not force and not _stale():
        return LIB
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found: cannot build libgrl_b200.so")
    objdir = os.path.join(PKG, "build")
    os.makedirs(objdir, exist_ok=True)
    if _stamp() != _defines():
        force = True  # different defines: every object is stale
    objs, procs = [], []
    for src in sources():
        obj = os.path.join(objdir, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        if (not force and os.path.exists(obj) and os.path.getmtime(obj) > os.path.getmtime(src)
                and not any(os.path.getmtime(h) > os.path.getmtime(obj)
                            for h in glob.glob(os.path.join(CSRC, "*.h")) + glob.glob(os.path.join(CSRC, "*.cuh"))
                            + [os.path.join(os.path.dirname(PKG), "include", "grl_b200.h")])):
            continue
        cmd = [nvcc] + NVCC_FLAGS + _defines().split() + ["-c", src, "-o", obj]  # A/B builds
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}:\n{out}")
        if verbose:
            sys.stderr.write(out)
        with open(os.path.join(objdir, os.path.basename(src)[:-3] + ".ptxas.log"), "w") as f:
            f.write(out)
    cmd = [nvcc, "-shared", "-o", LIB + ".tmp"] + objs
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}")
    os.replace(LIB + ".tmp", LIB)
    with open(STAMP, "w") as f:
        f.write(_defines())
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
