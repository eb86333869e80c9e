"""Builds libqagnn_b200.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100)."""
import glob
import hashlib
import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIBNAME = "libqagnn_b200.so"

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + ["-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-v",
]


def _nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def _sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def _stamp():
    h = hashlib.sha256()
    for p in _sources() + sorted(glob.glob(os.path.join(CSRC, "*.cuh"))) + [os.path.join(HERE, "..", "include", "qagnn_b200.h"), __file__]:
        with open(p, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def lib_path():
    return os.path.join(LIBDIR, LIBNAME)


def is_current():
    """True when the in-tree library was built from the current sources."""
    stamp_file = lib_path() + ".stamp"
    return os.path.exists(lib_path()) and os.path.exists(stamp_file) and open(stamp_file).read() == _stamp()


def build(force=False, verbose=False):
    """Compile every .cu under csrc/ into one shared library.  Returns its path."""
    os.makedirs(LIBDIR, exist_ok=True)
    out = lib_path()
    stamp_file = out + ".stamp"
    stamp = _stamp()
    if not force and os.path.exists(out) and os.path.exists(stamp_file) and open(stamp_file).read() == stamp:
        return out
    objs = []
    objdir = os.path.join(LIBDIR, "obj")
    os.makedirs(objdir, exist_ok=True)
    procs = []
    for src in _sources():
        obj = os.path.join(objdir, os.path.basename(src)[:-3] + ".o")
        cmd = [_nvcc(), "-c", src, "-o", obj] + [f for f in NVCC_FLAGS if f]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    log = []
    for src, p in procs:
        o, _ = p.communicate()
        log.append(f"== {os.path.basename(src)}\n{o}")
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}:\n{o}")
    cmd = [_nvcc(), "-shared", "-o", out] + objs + ARCH
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n" + r.stdout)
    with open(os.path.join(LIBDIR, "build.log"), "w") as f:
        f.write("\n".join(log))
    with open(stamp_file, "w") as f:
        f.write(stamp)
    if verbose:
        print("\n".join(log))
    return out


if __name__ == "__main__":
    print(build(force=True, verbose=True))
