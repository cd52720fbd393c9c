"""Builds libpulse_b200.so (all CUDA kernels + the C ABI) in-tree with nvcc for sm_90a (H100).

`python -m pulse_b200.build` or `__graft_entry__.build()`.  nvcc cross-compiles without a GPU.
The .so and the object files are build products (git-ignored); a fresh checkout builds them.
"""
import glob
import os
import shutil
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
LIB = os.path.join(PKG, "libpulse_b200.so")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]


def _nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found (set NVCC or add /usr/local/cuda/bin to PATH)")


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = sources() + glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(CSRC, "*.inc")) + glob.glob(os.path.join(ROOT, "include", "*.h"))
    return any(os.path.getmtime(p) > t for p in deps)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    objs = []
    obj_dir = os.path.join(PKG, "build")
    os.makedirs(obj_dir, exist_ok=True)
    common = [_nvcc(), *ARCH, "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC", "-I" + os.path.join(ROOT, "include"), "-I" + CSRC]
    if verbose:
        common += ["-Xptxas", "-v"]
    procs = []
    for src in sources():
        obj = os.path.join(obj_dir, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        hdr_t = max([os.path.getmtime(p) for p in glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(CSRC, "*.inc"))
                     + glob.glob(os.path.join(ROOT, "include", "*.h"))] + [0])
        if not force and os.path.exists(obj) and os.path.getmtime(obj) > max(os.path.getmtime(src), hdr_t):
            continue
        procs.append((src, subprocess.Popen(common + ["-c", src, "-o", obj], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for src, p in procs:
        out, _ = p.communicate()
        if verbose and out:
            print(out)
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}:\n{out}")
    link = [_nvcc(), *ARCH, "--shared", "-o", LIB, *objs, "-lcudart"]
    r = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
