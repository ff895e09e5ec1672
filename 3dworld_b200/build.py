"""Builds lib3dworld_b200.so (hand-written sm_90a CUDA + the extern "C" boundary of include/tw3d.h) in-tree with nvcc.
-fmad=false: the reference CPU path is built without FMA contraction (makefile:11, no -march); fused multiply-adds are written
explicitly (__fmaf_rn) only where they are provably bit-identical (see csrc/tw_noise.cuh)."""
import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "lib3dworld_b200.so")
SOURCES = ["tw_api.cu", "tw_heightgen.cu", "tw_erosion.cu", "tw_voxel.cu", "tw_streaming.cu", "tw_tiles.cu", "tw_multi.cu", "tw_voxel_post.cu", "tw_shadows.cu", "tw_tileset.cu", "tw_host.cpp"]
# device code the library loads at run time (cudaLibraryLoadFromFile), each built as <name>.cubin beside the library: the change list of a voxel model
# edit, the batch of small voxel grids and the batch of small voxel models (tw_voxel_post.cu loads them), and the AO map of heightmap tiles (tw_api.cu)
MODULES = ["tw_voxel_changes.cu", "tw_voxel_batch.cu", "tw_voxel_model_batch.cu", "tw_hmap_ao.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-fmad=false", "-prec-div=true", "-prec-sqrt=true",
              "-Xcompiler", "-fPIC,-ffp-contract=off,-fno-fast-math,-fvisibility=hidden", "--use_fast_math=false"]


def nvcc():
    for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def module_path(lib, src):
    return os.path.join(os.path.dirname(lib), src.rsplit(".", 1)[0] + ".cubin")


def needs_build():
    if not os.path.exists(LIB) or not all(os.path.exists(module_path(LIB, m)) for m in MODULES):
        return True
    t = min([os.path.getmtime(LIB)] + [os.path.getmtime(module_path(LIB, m)) for m in MODULES])
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "tw3d.h"), __file__]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False, lib=None, objdir=None):
    """lib / objdir (or TW_BUILD_LIB / TW_BUILD_OBJDIR): build a variant somewhere else without touching the shipped library (tools/ab_variants.sh)."""
    lib = lib or os.environ.get("TW_BUILD_LIB") or LIB
    if lib == LIB and not force and not needs_build():
        return LIB
    objdir = objdir or os.environ.get("TW_BUILD_OBJDIR") or os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    objs = []
    procs = []
    flags = [f for f in NVCC_FLAGS if f != "--use_fast_math=false"] + os.environ.get("TW_EXTRA_NVCC_FLAGS", "").split()
    for src in SOURCES:
        obj = os.path.join(objdir, src.rsplit(".", 1)[0] + ".o")
        cmd = [nvcc()] + flags + (["-Xptxas", "-v"] if verbose else []) + ["-x", "cu", "-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    for src in MODULES:
        cmd = [nvcc()] + flags + (["-Xptxas", "-v"] if verbose else []) + ["-cubin", os.path.join(CSRC, src), "-o", module_path(lib, src) + ".tmp"]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for src, p in procs:
        out, _ = p.communicate()
        if verbose and out:
            print(out)
        if p.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s" % (src, out))
    cmd = [nvcc(), "-shared", "-Wno-deprecated-gpu-targets", "-o", lib + ".tmp"] + objs + ["-Xlinker", "--no-undefined", "-lcudart_static", "-lpthread", "-ldl", "-lrt"]
    subprocess.check_call(cmd)
    for src in MODULES:
        os.replace(module_path(lib, src) + ".tmp", module_path(lib, src))
    os.replace(lib + ".tmp", lib)   # atomic: a concurrent snapshot of the tree never sees a half-written library
    return lib


if __name__ == "__main__":
    import sys
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
