"""In-tree build of the CUDA library: nvcc -> sgformer_b200/lib/libsgformer_b200.so (sm_90a only).

The .so is git-ignored and built by `__graft_entry__.build()`; nothing is JIT-compiled at run time."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB_DIR = os.path.join(HERE, "lib")
OBJ_DIR = os.path.join(HERE, "build", "obj")
LIB_PATH = os.path.join(LIB_DIR, "libsgformer_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]
CFLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC",
          "--expt-relaxed-constexpr"]


def _sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _deps_mtime():
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hdrs.append(os.path.join(os.path.dirname(HERE), "include", "sgformer_b200.h"))
    return max(os.path.getmtime(h) for h in hdrs)


def needs_build():
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    return any(os.path.getmtime(s) > t for s in _sources()) or _deps_mtime() > t


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB_PATH
    os.makedirs(LIB_DIR, exist_ok=True)
    os.makedirs(OBJ_DIR, exist_ok=True)
    hdr_t = _deps_mtime()

    def compile_one(src):
        obj = os.path.join(OBJ_DIR, os.path.basename(src)[:-3] + ".o")
        if not force and os.path.exists(obj) and os.path.getmtime(obj) > max(os.path.getmtime(src), hdr_t):
            return obj
        cmd = [NVCC] + ARCH_FLAGS + CFLAGS + ["-c", src, "-o", obj]
        if verbose:
            print(" ".join(cmd), file=sys.stderr)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        return obj

    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        objs = list(ex.map(compile_one, _sources()))
    cmd = [NVCC] + ARCH_FLAGS + ["-shared", "-o", LIB_PATH] + objs
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB_PATH


def build_variant(name, extra_flags, only=("spmm.cu",)):
    """Tuning aid: libsgformer_b200_<name>.so with `extra_flags` (e.g. ["-DSGF_SPMM_UNROLL=8"]) applied to the sources in
    `only`; all other objects are shared with the main build.  Load it with scripts/bench_*.py --lib."""
    build()
    vdir = os.path.join(OBJ_DIR, name)
    os.makedirs(vdir, exist_ok=True)
    objs = []
    for src in _sources():
        base = os.path.basename(src)
        if base in only:
            obj = os.path.join(vdir, base[:-3] + ".o")
            r = subprocess.run([NVCC] + ARCH_FLAGS + CFLAGS + list(extra_flags) + ["-c", src, "-o", obj], capture_output=True, text=True)
            if r.returncode != 0:
                raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        else:
            obj = os.path.join(OBJ_DIR, base[:-3] + ".o")
        objs.append(obj)
    out = os.path.join(LIB_DIR, f"libsgformer_b200_{name}.so")
    r = subprocess.run([NVCC] + ARCH_FLAGS + ["-shared", "-o", out] + objs, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return out


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
