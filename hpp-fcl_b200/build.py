"""In-tree build of the CUDA extension (sm_90a only: H100) with nvcc.

The product is a plain C-ABI shared library (include/hppfcl_b200.h): no torch
types cross the boundary, so it is built with nvcc directly rather than through
torch.utils.cpp_extension.
"""
import os
import shutil
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(_HERE, "csrc")
_SO = os.path.join(_HERE, "libhppfcl_b200.so")

GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]

NVCC_FLAGS = GENCODE + [
    "-O3", "-std=c++17", "-lineinfo",
    # bit-exact parity with the FP64 reference semantics: no FMA contraction
    # (the oracle is compiled -ffp-contract=off); fp64 div/sqrt are IEEE already.
    "-fmad=false",
    "-Xcompiler", "-fPIC", "-shared",
    "-Xptxas", "-v",
]


def library_path():
    return _SO


def _nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def sources():
    return sorted(os.path.join(_CSRC, f) for f in os.listdir(_CSRC) if f.endswith(".cu"))


def _deps():
    out = []
    for root, _, files in os.walk(_CSRC):
        out += [os.path.join(root, f) for f in files if f.endswith((".cu", ".cuh", ".h"))]
    out.append(os.path.join(_HERE, "..", "include", "hppfcl_b200.h"))
    return out


def build_extension(force=False, verbose=False):
    """Compile csrc/*.cu -> libhppfcl_b200.so (cross-compiles without a GPU).  Every translation unit is
    compiled on its own (in parallel: the big ones take a minute each) and the objects are linked into one
    shared library; device code never calls across units, so no relocatable device code is needed."""
    if not force and os.path.exists(_SO):
        t = os.path.getmtime(_SO)
        if all(os.path.getmtime(d) <= t for d in _deps()):
            return _SO
    from concurrent.futures import ThreadPoolExecutor
    objdir = os.path.join(_HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    ccbin = ["-ccbin", "/usr/bin/g++"] if os.path.exists("/usr/bin/g++") else []
    # the image exports CXX=/opt/gcc/bin/g++ (a wrapper); nvcc wants the system host compiler
    inc = ["-I", os.path.join(_HERE, "..", "include"), "-I", _CSRC]
    cflags = [f for f in NVCC_FLAGS if f != "-shared"]
    hdr_t = max(os.path.getmtime(d) for d in _deps() if not d.endswith(".cu"))

    def compile_one(src):
        obj = os.path.join(objdir, os.path.basename(src)[:-3] + ".o")
        if not force and os.path.exists(obj) and os.path.getmtime(obj) >= max(hdr_t, os.path.getmtime(src)):
            return obj, 0, "(up to date) " + obj + "\n"
        cmd = [_nvcc()] + cflags + ccbin + inc + ["-c", "-o", obj, src]
        res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        return obj, res.returncode, " ".join(cmd) + "\n" + res.stdout

    with ThreadPoolExecutor(max_workers=max(1, min(8, os.cpu_count() or 1))) as ex:
        results = list(ex.map(compile_one, sources()))
    out = "".join(r[2] for r in results)
    rc = max(r[1] for r in results)
    if rc == 0:
        cmd = [_nvcc()] + GENCODE + ["-shared", "-Xcompiler", "-fPIC"] + ccbin + \
              ["-o", _SO] + [r[0] for r in results]
        res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        out += " ".join(cmd) + "\n" + res.stdout
        rc = res.returncode
    log = os.path.join(_HERE, "build.log")
    with open(log, "w") as f:
        f.write(out)
    if verbose or rc != 0:
        print(out)
    if rc != 0:
        raise RuntimeError("nvcc failed (see %s)" % log)
    return _SO
