"""Builds hydragnn_b200/csrc/libhgb.so with nvcc for sm_90a (H100), in-tree next to the sources, so the package
imports from the repository without an install step.  No torch dependency: the library is a plain C-ABI shared object.
"""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(CSRC, "libhgb.so")
ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH_FLAGS + ["-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]


def _nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    raise RuntimeError("nvcc not found")


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _stamp():
    h = hashlib.sha256()
    for f in sorted(os.listdir(CSRC)) + ["../../include/hgb.h"]:
        if f.endswith((".cu", ".cuh", ".h")):
            h.update(open(os.path.join(CSRC, f), "rb").read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def _ensure_generated():
    """hgb_mace_gen.cuh is generated from hydragnn_b200/e3.py and committed; regenerate it only if it is missing."""
    if not os.path.exists(os.path.join(CSRC, "hgb_mace_gen.cuh")):
        sys.path.insert(0, CSRC)
        try:
            import gen_mace
            gen_mace.generate()
        finally:
            sys.path.pop(0)


def build(force=False, verbose=False):
    _ensure_generated()
    stamp_file = os.path.join(CSRC, ".build_stamp")
    stamp = _stamp()
    if not force and os.path.exists(LIB) and os.path.exists(stamp_file) and open(stamp_file).read() == stamp:
        return LIB
    nvcc = _nvcc()
    objs = []
    procs = []
    for src in sources():
        obj = os.path.join(CSRC, src[:-3] + ".o")
        cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            sys.stderr.write("nvcc failed on %s:\n%s\n" % (src, out))
        elif verbose:
            sys.stderr.write(out)
    if failed:
        raise RuntimeError("libhgb.so build failed")
    subprocess.check_call([nvcc, "-shared", "-o", LIB] + objs + ARCH_FLAGS + ["-lcudart_static", "-Xcompiler", "-fPIC"])
    open(stamp_file, "w").write(stamp)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
