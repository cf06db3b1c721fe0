"""Build libdreammat_b200.so (sm_90a only) in-tree with nvcc.

The shared object is the product's C-ABI (include/dreammat_b200.h); it lives next to the
package so it travels with the repo snapshot to the GPU box.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libdreammat_b200.so")
OBJDIR = os.path.join(HERE, "build")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-v",
]


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(LIBDIR, exist_ok=True)
    os.makedirs(OBJDIR, exist_ok=True)
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cuh")]
    hdrs.append(os.path.join(HERE, "..", "include", "dreammat_b200.h"))
    hdr_m = max(os.path.getmtime(h) for h in hdrs)
    objs, procs = [], []
    for s in sources():
        src = os.path.join(CSRC, s)
        obj = os.path.join(OBJDIR, s[:-3] + ".o")
        objs.append(obj)
        if force or not os.path.exists(obj) or os.path.getmtime(obj) < max(os.path.getmtime(src), hdr_m):
            cmd = ["nvcc", *NVCC_FLAGS, "-c", src, "-o", obj]
            procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for s, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            sys.stderr.write(f"--- nvcc failed for {s}\n{out}\n")
        else:
            with open(os.path.join(OBJDIR, s[:-3] + ".ptxas.log"), "w") as f:
                f.write(out)
            if verbose:
                print(out)
    if failed:
        raise RuntimeError("nvcc build failed")
    if procs or force or not os.path.exists(LIB):
        cmd = ["nvcc", "-shared", "-o", LIB, *objs, "-gencode", "arch=compute_90a,code=sm_90a", "-lcudart"]
        subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
