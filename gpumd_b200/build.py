"""Build libb200md.so (hand-written CUDA for sm_90a) in-tree with nvcc.

    python -m gpumd_b200.build          # or gpumd_b200.build.build_lib()

The shared library lands at gpumd_b200/libb200md.so (git-ignored, travels to the GPU box with the
gpurun snapshot).  nvcc cross-compiles without a GPU.
"""
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
LIB = PKG / "libb200md.so"
OBJ = PKG / "build"

CU_SOURCES = ["b2_host.cu", "b2_neighbor.cu", "b2_nep.cu", "b2_md.cu", "b2_tersoff.cu", "b2_eam.cu",
              "b2_tc_test.cu", "b2_stochastic.cu", "b2_measure.cu", "b2_nemd.cu", "b2_correlate.cu",
              "b2_minimize.cu", "b2_phonon.cu", "b2_rdf.cu"]
CPP_SOURCES = ["b2_nep_model.cpp"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC",
]


def _nvcc():
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(exe):
        raise RuntimeError("nvcc not found: libb200md cannot be built (there is no CPU fallback)")
    return exe


def _stale(target, deps):
    if not target.exists():
        return True
    t = target.stat().st_mtime
    return any(d.stat().st_mtime > t for d in deps)


def build_lib(force=False, verbose=False, variant=None, defs=()):
    """variant / defs: a diagnostic build with extra -D flags -> gpumd_b200/libb200md_<variant>.so
    (objects under build_<variant>/); selected at run time with B200MD_LIB=<path> (lib.py)."""
    if variant:
        return _build_lib(PKG / f"libb200md_{variant}.so", PKG / f"build_{variant}",
                          [f"-D{d}" for d in defs], force, verbose)
    return _build_lib(LIB, OBJ, [], force, verbose)


def _build_lib(LIB, OBJ, extra, force, verbose):
    nvcc = _nvcc()
    OBJ.mkdir(exist_ok=True)
    headers = list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.h")) + [PKG.parent / "include" / "b200md.h"]
    jobs = []
    objs = []
    for src in CU_SOURCES + CPP_SOURCES:
        s = CSRC / src
        o = OBJ / (s.stem + ".o")
        objs.append(o)
        if force or _stale(o, [s] + headers):
            jobs.append([nvcc] + NVCC_FLAGS + extra + ["-c", str(s), "-o", str(o)])

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + r.stdout + r.stderr)
        if verbose and (r.stdout or r.stderr):
            print(r.stdout + r.stderr)

    with ThreadPoolExecutor(max_workers=4) as ex:
        list(ex.map(run, jobs))
    if force or jobs or not LIB.exists():
        run([nvcc, "-shared", "-Xcompiler", "-fPIC", "-gencode", "arch=compute_90a,code=sm_90a",
             "-o", str(LIB)] + [str(o) for o in objs] + ["-lcudart"])
    return LIB


MGPU = PKG / "libb200md_mgpu.so"


def build_mgpu(force=False):
    """The multi-GPU domain module (csrc/b2_mgpu.cu: C++ host + CUDA + NCCL over the libb200md
    C-ABI) -> gpumd_b200/libb200md_mgpu.so."""
    nvcc = _nvcc()
    src = CSRC / "b2_mgpu.cu"
    deps = [src, PKG.parent / "include" / "b200md.h", PKG.parent / "include" / "b200md_mgpu.h", LIB]
    if force or _stale(MGPU, deps):
        cmd = [nvcc] + NVCC_FLAGS + ["-shared", str(src), "-o", str(MGPU), "-L" + str(PKG), "-lb200md",
                                     "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN", "-lnccl", "-lcudart"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("mgpu build failed:\n" + r.stdout + r.stderr)
    return MGPU


HOST = PKG / "host"
EXE = PKG / "b200md"


def build_host(force=False):
    """The C++ host layer (adapter classes + standalone driver) -> gpumd_b200/b200md."""
    nvcc = _nvcc()
    srcs = [HOST / f for f in ("potential.cpp", "force.cpp", "ensemble.cpp", "measure.cpp", "minimize.cpp",
                                       "phonon.cpp", "run.cpp")]
    deps = srcs + list(HOST.glob("*.h")) + [PKG.parent / "include" / "b200md.h", LIB]
    if force or _stale(EXE, deps):
        cmd = [nvcc, "-O2", "-std=c++17", "-x", "cu", "-gencode", "arch=compute_90a,code=sm_90a"] + \
            [str(s) for s in srcs] + ["-o", str(EXE), "-L" + str(PKG), "-lb200md",
                                      "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN", "-lcudart"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("host build failed:\n" + r.stdout + r.stderr)
    return EXE


GOLDEN = PKG.parent / "tests" / "golden"


def unpack_fixtures():
    """Test and benchmark inputs stored gzip-compressed under tests/golden/ (files in the repository
    stay below 1 MB) -> the plain-text file next to each one."""
    import gzip
    for gz in GOLDEN.glob("*.gz"):
        out = gz.with_suffix("")
        if _stale(out, [gz]):
            tmp = out.with_name(out.name + ".tmp")
            tmp.write_bytes(gzip.decompress(gz.read_bytes()))
            tmp.replace(out)
    return GOLDEN


if __name__ == "__main__":
    print(build_lib(force="--force" in sys.argv, verbose=True))
    print(build_mgpu(force="--force" in sys.argv))
    print(build_host(force="--force" in sys.argv))
    print(unpack_fixtures())
