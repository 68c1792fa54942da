"""In-tree build of the CUDA backend -> rav1e_b200/libb200rdo.so (sm_90a only).

nvcc cross-compiles without a GPU.  Objects go to build/ (git-ignored); the .so stays in
the package directory so it travels to the GPU box with the gpurun snapshot.
"""
import concurrent.futures as cf
import os
import shutil
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
OBJ = os.path.join(ROOT, "build", "obj")
LIB = os.path.join(PKG, "libb200rdo.so")
NVCC = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
HOSTCXX = "/usr/bin/g++"
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC,-Wall,-Wno-unused-function,-Wno-unknown-pragmas",
         "-ccbin", HOSTCXX, "--expt-relaxed-constexpr"]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _deps_mtime():
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hdrs.append(os.path.join(ROOT, "include", "b200rdo.h"))
    return max(os.path.getmtime(h) for h in hdrs)


def _compile(src, verbose):
    obj = os.path.join(OBJ, os.path.basename(src)[:-3] + ".o")
    if os.path.exists(obj) and os.path.getmtime(obj) > max(os.path.getmtime(src), _deps_mtime()):
        return obj, ""
    cmd = [NVCC, *ARCH, *FLAGS, "-c", src, "-o", obj]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
    return obj, r.stderr


def build(verbose=False, force=False):
    os.makedirs(OBJ, exist_ok=True)
    if force:
        for f in os.listdir(OBJ):
            os.remove(os.path.join(OBJ, f))
    srcs = sources()
    logs = []
    with cf.ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        results = list(ex.map(lambda s: _compile(s, verbose), srcs))
    objs = [o for o, _ in results]
    logs = [l for _, l in results if l]
    if (not os.path.exists(LIB)) or any(os.path.getmtime(o) > os.path.getmtime(LIB) for o in objs):
        cmd = [NVCC, *ARCH, "-shared", "-ccbin", HOSTCXX, "-o", LIB, *objs, "-lcudart_static",
               "-lpthread", "-ldl", "-lrt"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB, "\n".join(logs)


if __name__ == "__main__":
    lib, log = build(verbose="-v" in sys.argv, force="-f" in sys.argv)
    if log:
        print(log)
    print(lib)
