"""In-tree nvcc build of libodise_b200.so (sm_90a only) and of the C oracle.

Used by __graft_entry__.build(); no torch extension machinery: the product is a plain C-ABI shared library
(include/odise_b200.h) loaded with ctypes."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "odise_b200", "csrc")
OUT = os.path.join(ROOT, "odise_b200", "libodise_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC", "-I", os.path.join(ROOT, "include"), "-I", CSRC,
    "--expt-relaxed-constexpr", "-Xptxas", "-v",
]


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _needs_build(objs, srcs):
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(ROOT, "include", "odise_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    srcs = sources()
    objdir = os.path.join(ROOT, "build", "obj")
    os.makedirs(objdir, exist_ok=True)
    objs = [os.path.join(objdir, s[:-3] + ".o") for s in srcs]
    if not force and not _needs_build(objs, srcs):
        return OUT

    def compile_one(pair):
        src, obj = pair
        cmd = [NVCC, *FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        return src, r

    with ThreadPoolExecutor(max_workers=8) as ex:
        results = list(ex.map(compile_one, zip(srcs, objs)))
    log = []
    for src, r in results:
        log.append(f"== {src}\n{r.stderr}")
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError(f"nvcc failed on {src}")
    with open(os.path.join(ROOT, "build", "ptxas.log"), "w") as f:
        f.write("\n".join(log))
    if verbose:
        print("\n".join(log))
    r = subprocess.run([NVCC, "-shared", "-o", OUT, *objs, "-lcudart"], capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("link failed")
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
