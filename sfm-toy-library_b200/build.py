"""Builds libsfmb200.so (the C-ABI product, include/sfmb200.h) in-tree with nvcc for sm_90a (H100).

    python sfm-toy-library_b200/build.py            # incremental
    python sfm-toy-library_b200/build.py --force

nvcc cross-compiles without a GPU; the .so lands in sfm-toy-library_b200/lib/ (git-ignored build product).
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIBDIR = os.path.join(HERE, "lib")
SO = os.path.join(LIBDIR, "libsfmb200.so")
SOURCES = ["ctx.cu", "comm.cu", "match.cu", "match_tc.cu", "triangulate.cu", "ba.cu", "ransac.cu", "essential.cu", "homography.cu", "orb.cu", "jpeg.cu", "resize.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
HOST_CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC,-O3",
         "-ccbin", HOST_CXX, "--expt-relaxed-constexpr", "-Xptxas", "-v"]


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True); os.makedirs(LIBDIR, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(os.path.dirname(HERE), "include", "sfmb200.h"))
    headers.append(os.path.abspath(__file__))
    jobs = []
    for s in SOURCES:
        src = os.path.join(CSRC, s); obj = os.path.join(OBJ, s.replace(".cu", ".o"))
        if force or _stale(obj, [src] + headers):
            jobs.append((src, obj))

    def cc(job):
        src, obj = job
        r = subprocess.run([NVCC] + FLAGS + ["-c", src, "-o", obj], capture_output=True, text=True)
        return src, r
    with ThreadPoolExecutor(max_workers=len(jobs) or 1) as ex:
        for src, r in ex.map(cc, jobs):
            log = os.path.join(OBJ, os.path.basename(src) + ".log")
            with open(log, "w") as f:
                f.write(r.stdout + r.stderr)
            if r.returncode != 0:
                sys.stderr.write(r.stdout + r.stderr)
                raise RuntimeError(f"nvcc failed on {src}")
            if verbose:
                sys.stderr.write(r.stderr)
    objs = [os.path.join(OBJ, s.replace(".cu", ".o")) for s in SOURCES]
    if force or jobs or _stale(SO, objs):
        r = subprocess.run([NVCC, "-shared", "-o", SO] + objs + ["-ccbin", HOST_CXX, "-cudart", "static", "-ldl", "-lpthread"],
                           capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("link failed")
    return SO


def build_host(force=False):
    """C++ host shim (host/shim.cpp: the reference's three stage functions over the C ABI) + its test binary."""
    hdir = os.path.join(HERE, "host"); out = os.path.join(hdir, "build", "test_shim")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    deps = [os.path.join(hdir, f) for f in ("shim.cpp", "test_shim.cpp", "sfmtoylib_b200.h", "cv_min.h")] + [SO]
    if force or _stale(out, deps):
        r = subprocess.run([HOST_CXX, "-std=c++17", "-O2", "-Wall", os.path.join(hdir, "shim.cpp"), os.path.join(hdir, "test_shim.cpp"),
                            "-I", hdir, "-L", LIBDIR, "-lsfmb200", "-Wl,-rpath,$ORIGIN/../../lib", "-lpthread", "-o", out],
                           capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("host shim build failed")
    return out


def build_host_essential(force=False):
    """The shim built with SFMB200_SHIM_ESSENTIAL (findCameraMatricesFromMatch on the device too) + its test binary."""
    hdir = os.path.join(HERE, "host"); out = os.path.join(hdir, "build", "test_shim_essential")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    deps = [os.path.join(hdir, f) for f in ("shim.cpp", "test_shim_essential.cpp", "sfmtoylib_b200.h", "cv_min.h")] + [SO]
    if force or _stale(out, deps):
        r = subprocess.run([HOST_CXX, "-std=c++17", "-O2", "-Wall", "-DSFMB200_SHIM_ESSENTIAL", os.path.join(hdir, "shim.cpp"),
                            os.path.join(hdir, "test_shim_essential.cpp"), "-I", hdir, "-L", LIBDIR, "-lsfmb200", "-Wl,-rpath,$ORIGIN/../../lib",
                            "-lpthread", "-o", out], capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("host shim (SFMB200_SHIM_ESSENTIAL) build failed")
    return out


def build_host_homography(force=False):
    """The shim built with SFMB200_SHIM_HOMOGRAPHY (findHomographyInliers on the device too) + its test binary."""
    hdir = os.path.join(HERE, "host"); out = os.path.join(hdir, "build", "test_shim_homography")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    deps = [os.path.join(hdir, f) for f in ("shim.cpp", "test_shim_homography.cpp", "sfmtoylib_b200.h", "cv_min.h")] + [SO]
    if force or _stale(out, deps):
        r = subprocess.run([HOST_CXX, "-std=c++17", "-O2", "-Wall", "-DSFMB200_SHIM_HOMOGRAPHY", os.path.join(hdir, "shim.cpp"),
                            os.path.join(hdir, "test_shim_homography.cpp"), "-I", hdir, "-L", LIBDIR, "-lsfmb200", "-Wl,-rpath,$ORIGIN/../../lib",
                            "-lpthread", "-o", out], capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("host shim (SFMB200_SHIM_HOMOGRAPHY) build failed")
    return out


def build_images(force=False):
    """sfmtoylib::readImages (host/sfm_images.cpp: the imread loop of setImagesDirectory over sfmb200_decode_jpeg_batch) + its driver."""
    hdir = os.path.join(HERE, "host"); out = os.path.join(hdir, "build", "test_images")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    deps = [os.path.join(hdir, f) for f in ("sfm_images.cpp", "sfm_images.h", "test_images.cpp", "sfmtoylib_b200.h", "cv_min.h")] + [SO]
    if force or _stale(out, deps):
        r = subprocess.run([HOST_CXX, "-std=c++17", "-O2", "-Wall", os.path.join(hdir, "sfm_images.cpp"), os.path.join(hdir, "test_images.cpp"),
                            "-I", hdir, "-L", LIBDIR, "-lsfmb200", "-Wl,-rpath,$ORIGIN/../../lib", "-lpthread", "-o", out],
                           capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("readImages build failed")
    return out


def build_glue(force=False):
    """Host glue of SURVEY.md 8(f-1) (host/sfm_glue.cpp: indexed find2D3DMatches / mergeNewPointCloud) + its test binary, which
    checks it against the naive restatement in oracle/host_glue_naive.hpp.  Pure C++, no GPU, no CUDA library."""
    hdir = os.path.join(HERE, "host"); out = os.path.join(hdir, "build", "test_glue")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    deps = [os.path.join(hdir, f) for f in ("sfm_glue.cpp", "sfm_glue.h", "test_glue.cpp", "sfmtoylib_b200.h", "cv_min.h")]
    deps.append(os.path.join(os.path.dirname(HERE), "oracle", "host_glue_naive.hpp"))
    if force or _stale(out, deps):
        r = subprocess.run([HOST_CXX, "-std=c++17", "-O2", "-Wall", os.path.join(hdir, "sfm_glue.cpp"), os.path.join(hdir, "test_glue.cpp"),
                            "-I", hdir, "-o", out], capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("host glue build failed")
    return out


def build_ply(force=False):
    """ASCII PLY writers of SURVEY.md 8(f-4) (host/sfm_ply.cpp) + the small driver the CPU test feeds scenes to."""
    hdir = os.path.join(HERE, "host"); out = os.path.join(hdir, "build", "test_ply")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    deps = [os.path.join(hdir, f) for f in ("sfm_ply.cpp", "sfm_ply.h", "test_ply.cpp", "sfmtoylib_b200.h", "cv_min.h")]
    if force or _stale(out, deps):
        r = subprocess.run([HOST_CXX, "-std=c++17", "-O2", "-Wall", os.path.join(hdir, "sfm_ply.cpp"), os.path.join(hdir, "test_ply.cpp"),
                            "-I", hdir, "-o", out], capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("PLY writer build failed")
    return out


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
    print(build_host(force="--force" in sys.argv))
    print(build_host_essential(force="--force" in sys.argv))
    print(build_host_homography(force="--force" in sys.argv))
    print(build_images(force="--force" in sys.argv))
    print(build_glue(force="--force" in sys.argv))
    print(build_ply(force="--force" in sys.argv))
