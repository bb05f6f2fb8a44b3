"""In-tree build of libposeidon252_b200.so (hand-written sm_90a CUDA + the C ABI).

    python -m poseidon252_b200.build            # regenerate tables/PTX header and compile
    python -m poseidon252_b200.build --check    # exit 0 iff the library is up to date

nvcc cross-compiles for sm_90a (H100) without a GPU; the .so is built in-tree
(poseidon252_b200/lib/), so the package imports straight from the repository tree.
"""
import os
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
LIB = os.path.join(PKG, "lib", "libposeidon252_b200.so")
SOURCES = [os.path.join(CSRC, f) for f in ("kernels.cu", "capi.cu")]
DEPS = SOURCES + [os.path.join(CSRC, f) for f in ("hades_device.cuh", "fr_ptx.cuh", "hades_tables.inc", "kernels.h",
                                                 "host_field.h", "jubjub_device.cuh")] + [os.path.join(ROOT, "include", "poseidon252_b200.h")]
GENERATORS = [os.path.join(ROOT, "tools", f) for f in ("gen_tables.py", "gen_field_ptx.py", "hades_model.py")]

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "-shared", "-Xptxas", "-v"]


def nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return "nvcc"


def up_to_date():
    if not os.path.exists(LIB):
        return False
    t = os.path.getmtime(LIB)
    return all(os.path.getmtime(p) <= t for p in DEPS + GENERATORS if os.path.exists(p))


def generate():
    for g in ("gen_tables.py", "gen_field_ptx.py"):
        subprocess.check_call([sys.executable, os.path.join(ROOT, "tools", g)], stdout=subprocess.DEVNULL)


def build(force=False, verbose=False):
    if not force and up_to_date():
        return LIB
    generate()
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    extra = os.environ.get("P252_NVCC_EXTRA", "").split()
    cmd = [nvcc()] + NVCC_FLAGS + extra + ["-o", LIB] + SOURCES + ["-ldl"]
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    log = os.path.join(PKG, "lib", "build.log")
    with open(log, "w") as f:
        f.write(" ".join(cmd) + "\n" + res.stdout)
    if verbose or res.returncode != 0:
        print(res.stdout)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed, see %s" % log)
    return LIB


if __name__ == "__main__":
    if "--check" in sys.argv:
        sys.exit(0 if up_to_date() else 1)
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
