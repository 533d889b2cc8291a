#!/usr/bin/env python
"""Builds oracle/_ref/: the REFERENCE's own TSDF kernels, compiled for sm_90a from the sources where they lie under
/root/reference, with a mechanical, behaviour-preserving compatibility patch applied to a scratch copy (the reference does
not compile under CUDA 12.9 as it is, SURVEY.md section 8c).  Nothing from the reference is copied into the repository; the
outputs are shared libraries under oracle/_ref/ (git-ignored, shipped to the GPU box by gpurun).

TEST INFRASTRUCTURE ONLY: loaded by tests/ (parity of our CUDA path against the reference's CUDA path on the same inputs) and
by scripts that time the reference kernels beside ours.

Patch list (each is a textual substitution on the scratch copy):
  1. FL/SiftGPU/cuda_SimpleMatrixUtil.h  : `matNxM<4,1>::operator float4()` explicit specialisation needs `template<>`.
  2. FL/SiftGPU/cudaUtil.h               : `__shfl_down/__shfl_xor(...)` -> `_sync(0xffffffff, ...)` (removed in CUDA 9+).
  3. FL/DepthSensing/CUDASceneRepHashSDF.cu : texture REFERENCES (removed in CUDA 12) -> plain global pointers;
     `tex2D(depthTextureRef, x, y)` -> `g_refDepth[y * g_refW + x]` (point sampling at integer in-range coordinates, which is
     all the kernels ever do); `bindInputDepthColorTextures` stores the pointers with cudaMemcpyToSymbol.
  4. CUDAConstant.cu and CUDASceneRepHashSDF.cu are compiled as ONE translation unit (the `extern __constant__` parameter blocks
     would otherwise need relocatable device code); the three parameter headers get the `#pragma once` they lack.
Two builds: libref_tsdf_fast.so (--use_fast_math, as the reference ships: FriedLiver.vcxproj:124) and libref_tsdf.so (IEEE).
Further outputs (see build_solver / build_siftmgr): libref_solver[_fast].so (bundle adjustment), libref_siftmgr[_fast].so (match-manager kernels),
libref_imageutil.so (image and trajectory kernels), and libref_kabsch_host.so -- the reference's host-callable Kabsch / eigen code compiled by
g++, which runs on the CPU; libref_sift_emulated.so -- the reference's SiftGPU (detection, matching) compiled by g++ against a CPU emulation
of CUDA (build_sift_emulated), which also runs on the CPU.
"""
import os
import re
import shutil
import subprocess
import sys

REF = "/root/reference/FriedLiver"
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")
TMP = "/tmp/bf_ref_build"


def patch(path, subs):
    s = open(path, encoding="latin-1").read()
    for pat, rep, count in subs:
        s, n = re.subn(pat, rep, s, flags=re.S)
        if count is not None and n != count:
            raise RuntimeError(f"{path}: pattern {pat!r} matched {n} times, expected {count}")
    open(path, "w", encoding="latin-1").write(s)


def main():
    if not os.path.isdir(REF):
        print("oracle/build_ref.py: /root/reference not present, nothing to do")
        return 0
    shutil.rmtree(TMP, ignore_errors=True)
    os.makedirs(TMP)
    os.makedirs(OUT, exist_ok=True)
    ds, sg = os.path.join(REF, "Source", "DepthSensing"), os.path.join(REF, "Source", "SiftGPU")
    for f in ("CUDAConstant.cu", "CUDASceneRepHashSDF.cu", "VoxelUtilHashSDF.h", "DepthCameraUtil.h", "CUDAHashParams.h",
              "CUDADepthCameraParams.h", "CUDARayCastParams.h"):
        shutil.copy(os.path.join(ds, f), TMP)
    for f in ("cuda_SimpleMatrixUtil.h", "cudaUtil.h"):
        shutil.copy(os.path.join(sg, f), TMP)
    patch(os.path.join(TMP, "cuda_SimpleMatrixUtil.h"),
          [(r"\ninline __device__ __host__ matNxM<4, 1>::operator float4\(\)", "\ntemplate<> inline __device__ __host__ matNxM<4, 1>::operator float4()", 1)])
    patch(os.path.join(TMP, "cudaUtil.h"),
          [(r"__shfl_down\(", "__shfl_down_sync(0xffffffffu, ", None), (r"__shfl_xor\(", "__shfl_xor_sync(0xffffffffu, ", None)])
    patch(os.path.join(TMP, "CUDASceneRepHashSDF.cu"), [
        (r"texture<float, cudaTextureType2D, cudaReadModeElementType> depthTextureRef;", "__device__ const float* g_refDepth; __device__ unsigned int g_refW;", 1),
        (r"texture<uchar4, cudaTextureType2D, cudaReadModeElementType> colorTextureRef;", "__device__ const uchar4* g_refColor;", 1),
        (r"cutilSafeCall\(cudaBindTexture2D\(0, depthTextureRef[^;]*;", "cutilSafeCall(cudaMemcpyToSymbol(g_refDepth, &depthCameraData.d_depthData, sizeof(float*))); cutilSafeCall(cudaMemcpyToSymbol(g_refW, &width, sizeof(unsigned int)));", 1),
        (r"cutilSafeCall\(cudaBindTexture2D\(0, colorTextureRef[^;]*;", "cutilSafeCall(cudaMemcpyToSymbol(g_refColor, &depthCameraData.d_colorData, sizeof(uchar4*)));", 1),
        (r"depthTextureRef\.filterMode = cudaFilterModePoint;", "", 1),
        (r"colorTextureRef\.filterMode = cudaFilterModePoint;", "", 1),
        (r"tex2D\(depthTextureRef,\s*([^,()]+),\s*([^,()]+)\)", r"g_refDepth[(\2) * g_refW + (\1)]", None),
        (r"tex2D\(colorTextureRef,\s*([^,()]+),\s*([^,()]+)\)", r"g_refColor[(\2) * g_refW + (\1)]", None),
    ])
    for f in ("CUDAHashParams.h", "CUDADepthCameraParams.h", "CUDARayCastParams.h"):      # no include guards in the reference
        q = os.path.join(TMP, f)
        open(q, "w", encoding="latin-1").write("#pragma once\n" + open(os.path.join(ds, f), encoding="latin-1").read())
    unit = os.path.join(TMP, "ref_tsdf_unit.cu")
    # definitions first; the headers' `extern __constant__` re-declarations are dropped (nvcc's host pass turns a __constant__
    # definition into a static shadow variable, which may not follow an extern declaration of the same name)
    patch(os.path.join(TMP, "VoxelUtilHashSDF.h"), [
        (r"extern\s+__constant__ HashParams c_hashParams;", "", 1),
        # `__align__(16)` placed BEFORE `struct` is honoured by MSVC (the reference's host compiler: sizeof(HashEntry) == 32) and
        # silently ignored by gcc / nvcc-on-Linux (20 bytes) -- and then the reference's own 8-byte entry copies (operator=,
        # VoxelUtilHashSDF.h:70-72) fault with "misaligned address".  Put the attribute where every compiler honours it.
        (r"__align__\(16\)\s*struct HashEntry", "struct __align__(16) HashEntry", 1)])
    patch(os.path.join(TMP, "DepthCameraUtil.h"), [(r"extern __constant__ DepthCameraParams c_depthCameraParams;", "", 1)])
    open(unit, "w").write('#include "CUDAConstant.cu"\n#include "CUDASceneRepHashSDF.cu"\n')
    inc = ["-I", TMP, "-I", os.path.join(REF, "Include", "cutil", "inc")]
    base = ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-w", "-shared", "-Xcompiler", "-fPIC", "-Xlinker", "-Bsymbolic",
            "-Xcompiler", "-fpermissive"] + inc
    for name, extra in (("libref_tsdf_fast.so", ["--use_fast_math"]), ("libref_tsdf.so", [])):
        cmd = base + extra + [unit, "-o", os.path.join(OUT, name), "-lcudart"]
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout[-4000:])
            raise RuntimeError(f"building {name} failed")
    build_solver()
    build_siftmgr()
    build_sift_emulated()
    build_mgr_emulated()
    build_fuse_emulated()
    build_trajectory_host()
    build_raycast_emulated()
    build_sens_host()
    build_marchingcubes_emulated()
    build_mesh_host()
    build_sensordata_host()
    print("oracle/_ref built:", sorted(os.listdir(OUT)))
    return 0


def build_solver():
    """The reference's bundle-adjustment solver (FL/Solver/SolverBundling.cu + FL/SBA.cu) for sm_90a -> libref_solver[_fast].so.
    Scratch tree mirrors the reference's relative include layout; patches: the two listed at the top (template<>, shfl_sync) plus
      5. FL/Solver/SolverBundlingUtil.h : `__shfl_down` -> `_sync`;
      6. FL/SBA.cu : the Windows back-slash in the LieDerivUtil.h include -> slash;
      7. stub headers standing in for <windows.h>, <conio.h> and mLib's core-base/common.h (MLIB_EXCEPTION / MLIB_ASSERT /
         SAFE_DELETE_ARRAY only -- CUDATimer.h and cudaUtil.h include them, the solver kernels use nothing from them)."""
    root = os.path.join(TMP, "solver")
    src = os.path.join(root, "Source")
    S = os.path.join(REF, "Source")
    for d in (os.path.join(src, "Solver"), os.path.join(src, "SiftGPU"), os.path.join(root, "SiftGPU"), os.path.join(root, "stubs", "core-base")):
        os.makedirs(d)
    for f in os.listdir(os.path.join(S, "Solver")):
        if f.endswith(".h") or f == "SolverBundling.cu":
            shutil.copy(os.path.join(S, "Solver", f), os.path.join(src, "Solver"))
    for f in ("SolverUtil.h", "GlobalDefines.h", "CUDACacheUtil.h", "CUDACameraUtil.h", "mLibCuda.h", "SBA.cu"):
        shutil.copy(os.path.join(S, f), src)
    for f in ("SIFTImageManager.h", "cuda_SimpleMatrixUtil.h", "cudaUtil.h", "CUDATimer.h"):
        for d in (os.path.join(src, "SiftGPU"), os.path.join(root, "SiftGPU")):       # "../SiftGPU/" and "../../SiftGPU/" includes
            shutil.copy(os.path.join(S, "SiftGPU", f), d)
    for d in (os.path.join(src, "SiftGPU"), os.path.join(root, "SiftGPU")):
        patch(os.path.join(d, "cuda_SimpleMatrixUtil.h"),
              [(r"\ninline __device__ __host__ matNxM<4, 1>::operator float4\(\)", "\ntemplate<> inline __device__ __host__ matNxM<4, 1>::operator float4()", 1)])
        patch(os.path.join(d, "cudaUtil.h"),
              [(r"__shfl_down\(", "__shfl_down_sync(0xffffffffu, ", None), (r"__shfl_xor\(", "__shfl_xor_sync(0xffffffffu, ", None)])
    patch(os.path.join(src, "Solver", "SolverBundlingUtil.h"),
          [(r"__shfl_down\(", "__shfl_down_sync(0xffffffffu, ", None), (r"__shfl_xor\(", "__shfl_xor_sync(0xffffffffu, ", None)])
    patch(os.path.join(src, "SBA.cu"), [(r'#include "Solver\\LieDerivUtil.h"', '#include "Solver/LieDerivUtil.h"', 1)])
    st = os.path.join(root, "stubs")
    open(os.path.join(st, "windows.h"), "w").write("#pragma once\n#include <mutex>\n#include <list>\n#include <string>\n#include <fstream>\n#include <algorithm>\n")
    open(os.path.join(st, "conio.h"), "w").write("#pragma once\n")
    open(os.path.join(st, "core-base", "common.h"), "w").write(
        "#pragma once\n#include <stdexcept>\n#include <string>\n#define MLIB_EXCEPTION(s) std::runtime_error(std::string(s))\n"
        "#define MLIB_ASSERT(x)\n#define SAFE_DELETE_ARRAY(p) { if (p) { delete[] (p); (p) = NULL; } }\n")
    base = ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-w", "-shared", "-Xcompiler", "-fPIC", "-Xlinker", "-Bsymbolic",
            "-Xcompiler", "-fpermissive", "-I", st, "-I", src, "-I", os.path.join(src, "SiftGPU"), "-I", os.path.join(src, "Solver"),
            "-I", os.path.join(REF, "Include", "cutil", "inc")]
    for name, extra in (("libref_solver_fast.so", ["--use_fast_math"]), ("libref_solver.so", [])):
        cmd = base + extra + [os.path.join(src, "Solver", "SolverBundling.cu"), os.path.join(src, "SBA.cu"), "-o", os.path.join(OUT, name), "-lcudart"]
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout[-4000:])
            raise RuntimeError(f"building {name} failed")


def build_siftmgr():
    """The reference's match-manager kernels (FL/SiftGPU/SIFTImageManager.cu: SortKeyPointMatchesCU, FilterKeyPointMatchesCU,
    FilterMatchesBySurfaceAreaCU, FilterMatchesByDenseVerifyCU, AddCurrToResidualsCU) for sm_90a -> libref_siftmgr[_fast].so, through
    oracle/ref_siftmgr_wrap.cu (our own C entry points, which includes the scratch copy as one translation unit).  Patches: template<>
    and shfl_sync as above, in every header that uses them; stub headers as for the solver."""
    root = os.path.join(TMP, "siftmgr")
    src = os.path.join(root, "Source")
    S = os.path.join(REF, "Source")
    for d in (os.path.join(src, "SiftGPU"), os.path.join(root, "stubs", "core-base")):
        os.makedirs(d)
    for f in os.listdir(os.path.join(S, "SiftGPU")):
        if f.endswith(".h") or f == "SIFTImageManager.cu":
            shutil.copy(os.path.join(S, "SiftGPU", f), os.path.join(src, "SiftGPU"))
    for f in ("GlobalDefines.h", "CUDACacheUtil.h", "mLibCuda.h"):
        shutil.copy(os.path.join(S, f), src)
    sg = os.path.join(src, "SiftGPU")
    patch(os.path.join(sg, "cuda_SimpleMatrixUtil.h"),
          [(r"\ninline __device__ __host__ matNxM<4, 1>::operator float4\(\)", "\ntemplate<> inline __device__ __host__ matNxM<4, 1>::operator float4()", 1)])
    for f in os.listdir(sg):
        patch(os.path.join(sg, f), [(r"__shfl_down\(", "__shfl_down_sync(0xffffffffu, ", None), (r"__shfl_xor\(", "__shfl_xor_sync(0xffffffffu, ", None)])
    st = os.path.join(root, "stubs")
    open(os.path.join(st, "windows.h"), "w").write("#pragma once\n#include <cfloat>\n#include <mutex>\n#include <list>\n#include <string>\n#include <fstream>\n#include <algorithm>\n")
    open(os.path.join(st, "conio.h"), "w").write("#pragma once\n")
    open(os.path.join(st, "core-base", "common.h"), "w").write(
        "#pragma once\n#include <stdexcept>\n#include <string>\ntypedef unsigned char uchar;\n#define MLIB_EXCEPTION(s) std::runtime_error(std::string(s))\n"
        "#define MLIB_ASSERT(x)\n#define SAFE_DELETE_ARRAY(p) { if (p) { delete[] (p); (p) = NULL; } }\n")
    base = ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-w", "-shared", "-Xcompiler", "-fPIC", "-Xlinker", "-Bsymbolic",
            "-Xcompiler", "-fpermissive", "-I", st, "-I", src, "-I", sg, "-I", os.path.join(REF, "Include", "cutil", "inc")]
    for name, extra in (("libref_siftmgr_fast.so", ["--use_fast_math"]), ("libref_siftmgr.so", [])):
        cmd = base + extra + [os.path.join(HERE, "ref_siftmgr_wrap.cu"), "-o", os.path.join(OUT, name), "-lcudart"]
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout[-6000:])
            raise RuntimeError(f"building {name} failed")
    # the reference's image kernels (rows a20 / a21) and trajectory kernels (row a22): FL/CUDAImageUtil.cu, FL/OnlineBundler.cu
    for f in ("CUDAImageUtil.cu", "CUDAImageUtil.h", "OnlineBundler.cu", "CUDACameraUtil.h"):
        shutil.copy(os.path.join(S, f), src)
    shutil.copy(os.path.join(S, "mLibCuda.h"), os.path.join(src, "mlibCuda.h"))          # `#include "mlibCuda.h"`: a case-insensitive file system is assumed
    cmd = base + [os.path.join(HERE, "ref_imageutil_wrap.cu"), "-o", os.path.join(OUT, "libref_imageutil.so"), "-lcudart"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout[-6000:])
        raise RuntimeError("building libref_imageutil.so failed")
    # the reference's host-callable Kabsch filter / eigen code, compiled by g++ (its `#ifdef __CUDACC__` picks `__host__` then): runs on the CPU
    cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
    cmd = ["g++", "-O2", "-w", "-fpermissive", "-ffp-contract=off", "-shared", "-fPIC", "-I", st, "-I", src, "-I", sg, "-I", os.path.join(REF, "Include", "cutil", "inc"),
           "-I", cuda_inc, os.path.join(HERE, "ref_kabsch_host.cpp"), "-o", os.path.join(OUT, "libref_kabsch_host.so"), "-lm"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout[-6000:])
        raise RuntimeError("building libref_kabsch_host.so failed")


def build_sift_emulated():
    """The reference's SiftGPU -- detection and descriptor matching, FL/SiftGPU/{ProgramCU.cu, SiftPyramid.cpp, SiftGPU.cpp, SiftMatch.cpp,
    CuTexImage.cpp, GlobalUtil.cpp, CUDASiftConstant.cu} -- compiled by g++ against a CPU emulation of CUDA (oracle/ref_emu/ref_emu_cuda.h on top of
    tests/cuda_emu/cuda_emu.h) -> libref_sift_emulated.so.  ProgramCU.cu is written against texture REFERENCES, which CUDA 12 removed, so nvcc
    cannot rebuild it here; emulated, the reference's own kernels run on the CPU and pin the SIFT oracles without a GPU.  Patches on the scratch copy:
      a. `kernel << <grid, block>> >(args)` -> `EMU_KERNEL(kernel, grid, block)(args)`;
      b. ComputeOrientation_Kernel: the barrier inside `if (tidx < 36)` becomes a barrier among those 36 threads, the barrier only thread 0 reaches
         is dropped, `weights[maxIndex]` is guarded for maxIndex == -1 (an out-of-bounds shared-memory store on the GPU, memory corruption on a host);
      c. ComputeDescriptor_Kernel: `des[8]` -> `des[9]` (the kernel indexes des[8] when an angle difference rounds to 8.0 bins);
      d. `(unsigned int)round(x)` of the four window extents -> the GPU's saturating conversion (a window outside the image has a negative extent:
         0 on the GPU, undefined behaviour in C++).
    None of them changes what the kernels compute."""
    root = os.path.join(TMP, "siftemu")
    src = os.path.join(root, "Source")
    S = os.path.join(REF, "Source")
    sg = os.path.join(src, "SiftGPU")
    os.makedirs(sg)
    for f in os.listdir(os.path.join(S, "SiftGPU")):
        if f.endswith((".h", ".cpp", ".cu")):
            shutil.copy(os.path.join(S, "SiftGPU", f), sg)
    for f in ("GlobalDefines.h", "CUDACacheUtil.h", "mLibCuda.h"):
        shutil.copy(os.path.join(S, f), src)
    patch(os.path.join(sg, "cuda_SimpleMatrixUtil.h"),
          [(r"\ninline __device__ __host__ matNxM<4, 1>::operator float4\(\)", "\ntemplate<> inline __device__ __host__ matNxM<4, 1>::operator float4()", 1)])
    launch = (r"([A-Za-z_]\w*(?:<[^<>()]*>)?)\s*<<\s*<\s*([^;]*?)\s*>>\s*>\s*\(", r"EMU_KERNEL(\1, \2)(", None)
    patch(os.path.join(sg, "ProgramCU.cu"), [
        launch,
        (r"(target\[tidx\] = \(source\[m\] \+ source\[c\] \+ source\[p\]\)\*one_third;\s*)__syncthreads\(\);", r"\1emu_sync_first(36);", 1),
        (r"weights\[maxIndex\] = -1\.0f;\s*__syncthreads\(\);", "if (maxIndex >= 0) weights[maxIndex] = -1.0f;", 1),
        (r"__shared__ float des\[8\];", "__shared__ float des[9];", 1),
        (r"\(unsigned int\)round\(([^;]*?)\);", r"emu_f2u(round(\1));", 4),
        (r"#if !\(COLMATCH_BLOCK_WIDTH == 32\)", "#if 1", 3),
    ])
    emu_dir = os.path.join(HERE, "ref_emu")
    cmd = ["g++", "-std=c++17", "-O2", "-w", "-fpermissive", "-ffp-contract=off", "-shared", "-fPIC", "-pthread", "-D__CUDACC__", "-x", "c++",
           "-I", emu_dir, "-I", os.path.join(os.path.dirname(HERE), "tests", "cuda_emu"), "-I", src, "-I", sg, "-I", os.path.join(REF, "Include", "cutil", "inc"),
           os.path.join(HERE, "ref_sift_emulated.cpp")]
    cmd += [os.path.join(sg, f) for f in ("ProgramCU.cu", "CUDASiftConstant.cu", "SiftPyramid.cpp", "SiftGPU.cpp", "SiftMatch.cpp", "CuTexImage.cpp", "GlobalUtil.cpp")]
    cmd += ["-o", os.path.join(OUT, "libref_sift_emulated.so"), "-lm"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout[-8000:])
        raise RuntimeError("building libref_sift_emulated.so failed")


def build_mgr_emulated():
    """The reference's match-manager, image and trajectory kernels (FL/SiftGPU/SIFTImageManager.cu, FL/CUDAImageUtil.cu, FL/OnlineBundler.cu) compiled
    by g++ against the CUDA emulation -> libref_mgr_emulated.so, through the same two wrapper files the GPU builds use (oracle/ref_siftmgr_wrap.cu,
    oracle/ref_imageutil_wrap.cu; their own launches are rewritten like the reference's).  Runs on the CPU: pins rows a19 - a22 without a GPU.
    __NVCC__ is defined so that cuda_svd3.h takes its device flavour of rsqrt (the emulation maps it to 1 / sqrtf, the oracle's default)."""
    root = os.path.join(TMP, "mgremu")
    src = os.path.join(root, "Source")
    S = os.path.join(REF, "Source")
    sg = os.path.join(src, "SiftGPU")
    os.makedirs(sg)
    for f in os.listdir(os.path.join(S, "SiftGPU")):
        if f.endswith(".h") or f == "SIFTImageManager.cu":
            shutil.copy(os.path.join(S, "SiftGPU", f), sg)
    for f in ("GlobalDefines.h", "CUDACacheUtil.h", "mLibCuda.h", "CUDAImageUtil.cu", "CUDAImageUtil.h", "OnlineBundler.cu", "CUDACameraUtil.h"):
        shutil.copy(os.path.join(S, f), src)
    shutil.copy(os.path.join(S, "mLibCuda.h"), os.path.join(src, "mlibCuda.h"))
    patch(os.path.join(sg, "cuda_SimpleMatrixUtil.h"),
          [(r"\ninline __device__ __host__ matNxM<4, 1>::operator float4\(\)", "\ntemplate<> inline __device__ __host__ matNxM<4, 1>::operator float4()", 1)])
    launch = (r"([A-Za-z_]\w*(?:<[^<>()]*>)?)\s*<<\s*<\s*([^;]*?)\s*>>\s*>\s*\(", r"EMU_KERNEL(\1, \2)(", None)
    for f in (os.path.join(sg, "SIFTImageManager.cu"), os.path.join(src, "CUDAImageUtil.cu"), os.path.join(src, "OnlineBundler.cu")):
        patch(f, [launch])
    units = []
    for w in ("ref_siftmgr_wrap.cu", "ref_imageutil_wrap.cu"):
        dst = os.path.join(root, w.replace(".cu", "_emu.cpp"))
        shutil.copy(os.path.join(HERE, w), dst)
        patch(dst, [launch])
        units.append(dst)
    emu_dir = os.path.join(HERE, "ref_emu")
    cmd = ["g++", "-std=c++17", "-O2", "-w", "-fpermissive", "-ffp-contract=off", "-shared", "-fPIC", "-pthread", "-D__CUDACC__", "-D__NVCC__",
           "-I", emu_dir, "-I", os.path.join(os.path.dirname(HERE), "tests", "cuda_emu"), "-I", src, "-I", sg, "-I", os.path.join(REF, "Include", "cutil", "inc")]
    cmd += units + ["-o", os.path.join(OUT, "libref_mgr_emulated.so"), "-lm"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout[-8000:])
        raise RuntimeError("building libref_mgr_emulated.so failed")


def build_fuse_emulated():
    """The reference's chunk -> keyframe fusion, host code of its manager class (FL/SiftGPU/SIFTImageManager.cpp: fuseToGlobal / computeTracks / findTrack), compiled with the
    class and its kernels (SIFTImageManager.cu) by g++ against the CUDA emulation -> libref_fuse_emulated.so (wrapper: oracle/ref_fuse_wrap.cpp).  Pins row N2's oracle
    (oracle/fuse_oracle.c) without a GPU.  The two application-state headers the .cpp includes (and uses only in comments) are empty files in the scratch tree."""
    root = os.path.join(TMP, "fuseemu")
    src = os.path.join(root, "Source")
    S = os.path.join(REF, "Source")
    sg = os.path.join(src, "SiftGPU")
    os.makedirs(sg)
    for f in os.listdir(os.path.join(S, "SiftGPU")):
        if f.endswith(".h") or f in ("SIFTImageManager.cu", "SIFTImageManager.cpp"):
            shutil.copy(os.path.join(S, "SiftGPU", f), sg)
    for f in ("GlobalDefines.h", "CUDACacheUtil.h", "mLibCuda.h"):
        shutil.copy(os.path.join(S, f), src)
    shutil.copy(os.path.join(S, "mLibCuda.h"), os.path.join(src, "mlibCuda.h"))
    for f in ("GlobalBundlingState.h", "GlobalAppState.h"):
        open(os.path.join(src, f), "w").write("#pragma once\n")
    patch(os.path.join(sg, "cuda_SimpleMatrixUtil.h"),
          [(r"\ninline __device__ __host__ matNxM<4, 1>::operator float4\(\)", "\ntemplate<> inline __device__ __host__ matNxM<4, 1>::operator float4()", 1)])
    launch = (r"([A-Za-z_]\w*(?:<[^<>()]*>)?)\s*<<\s*<\s*([^;]*?)\s*>>\s*>\s*\(", r"EMU_KERNEL(\1, \2)(", None)
    patch(os.path.join(sg, "SIFTImageManager.cu"), [launch])
    # the last member function of the file (fuseLocalKeyDepths, a debugging aid over mLib's DepthImage32) is cut; nothing on the path calls it
    patch(os.path.join(sg, "SIFTImageManager.cpp"), [(r"void SIFTImageManager::fuseLocalKeyDepths\(.*\Z", "", 1)])
    emu_dir = os.path.join(HERE, "ref_emu")
    cmd = ["g++", "-std=c++17", "-O2", "-w", "-fpermissive", "-ffp-contract=off", "-shared", "-fPIC", "-pthread", "-D__CUDACC__", "-D__NVCC__",
           "-I", emu_dir, "-I", os.path.join(os.path.dirname(HERE), "tests", "cuda_emu"), "-I", src, "-I", sg, "-I", os.path.join(REF, "Include", "cutil", "inc"),
           os.path.join(HERE, "ref_fuse_wrap.cpp"), "-o", os.path.join(OUT, "libref_fuse_emulated.so"), "-lm"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout[-8000:])
        raise RuntimeError("building libref_fuse_emulated.so failed")


def build_raycast_emulated():
    """The reference's ray-cast kernels (FL/DepthSensing/CUDARayCastSDF.cu with RayCastSDFUtil.h, VoxelUtilHashSDF.h, CUDAConstant.cu) compiled by g++ against
    the CUDA emulation -> libref_raycast_emulated.so (wrapper: oracle/ref_raycast_wrap.cu).  Runs on the CPU: pins row N3's oracle without a GPU and without
    Direct3D.  Patches on the scratch copies: launch syntax; renderCS binds its two interval textures to cudaArrays that Direct3D rendered -- here they are
    linear float images bound with cudaBindTexture2D; the HashEntry alignment attribute where gcc honours it (see main()); the matNxM specialisation."""
    root = os.path.join(TMP, "rcemu")
    os.makedirs(root)
    ds, sg = os.path.join(REF, "Source", "DepthSensing"), os.path.join(REF, "Source", "SiftGPU")
    for f in ("CUDAConstant.cu", "CUDARayCastSDF.cu", "RayCastSDFUtil.h", "VoxelUtilHashSDF.h", "DepthCameraUtil.h", "CUDAHashParams.h", "CUDADepthCameraParams.h", "CUDARayCastParams.h"):
        shutil.copy(os.path.join(ds, f), root)
    for f in ("cuda_SimpleMatrixUtil.h", "cudaUtil.h"):
        shutil.copy(os.path.join(sg, f), root)
    patch(os.path.join(root, "cuda_SimpleMatrixUtil.h"),
          [(r"\ninline __device__ __host__ matNxM<4, 1>::operator float4\(\)", "\ntemplate<> inline __device__ __host__ matNxM<4, 1>::operator float4()", 1)])
    for f in ("CUDAHashParams.h", "CUDADepthCameraParams.h", "CUDARayCastParams.h"):
        q = os.path.join(root, f)
        open(q, "w", encoding="latin-1").write("#pragma once\n" + open(os.path.join(ds, f), encoding="latin-1").read())
    patch(os.path.join(root, "VoxelUtilHashSDF.h"), [(r"__align__\(16\)\s*struct HashEntry", "struct __align__(16) HashEntry", 1)])
    # `-gradientForPoint(...)`: cutil_math's unary minus takes a non-const reference, which MSVC / nvcc bind to a temporary and g++ does not
    patch(os.path.join(root, "RayCastSDFUtil.h"), [(r"float3 normal = -gradientForPoint\(hash, currentIso\);", "float3 g_ = gradientForPoint(hash, currentIso); float3 normal = -g_;", 1)])
    launch = (r"([A-Za-z_]\w*(?:<[^<>()]*>)?)\s*<<\s*<\s*([^;]*?)\s*>>\s*>\s*\(", r"EMU_KERNEL(\1, \2)(", None)
    patch(os.path.join(root, "CUDARayCastSDF.cu"), [
        launch,
        (r"cudaBindTextureToArray\(rayMinTextureRef, rayCastData\.d_rayIntervalSplatMinArray, channelDesc\);",
         "cudaBindTexture2D(0, &rayMinTextureRef, (const void*)rayCastData.d_rayIntervalSplatMinArray, &channelDesc, rayCastParams.m_width, rayCastParams.m_height, rayCastParams.m_width * sizeof(float));", 1),
        (r"cudaBindTextureToArray\(rayMaxTextureRef, rayCastData\.d_rayIntervalSplatMaxArray, channelDesc\);",
         "cudaBindTexture2D(0, &rayMaxTextureRef, (const void*)rayCastData.d_rayIntervalSplatMaxArray, &channelDesc, rayCastParams.m_width, rayCastParams.m_height, rayCastParams.m_width * sizeof(float));", 1)])
    unit = os.path.join(root, "ref_raycast_wrap_emu.cpp")
    shutil.copy(os.path.join(HERE, "ref_raycast_wrap.cu"), unit)
    emu_dir = os.path.join(HERE, "ref_emu")
    cmd = ["g++", "-std=c++17", "-O2", "-w", "-fpermissive", "-ffp-contract=off", "-shared", "-fPIC", "-pthread", "-D__CUDACC__", "-D__NVCC__",
           "-I", emu_dir, "-I", os.path.join(os.path.dirname(HERE), "tests", "cuda_emu"), "-I", root, "-I", os.path.join(REF, "Include", "cutil", "inc"),
           unit, "-o", os.path.join(OUT, "libref_raycast_emulated.so"), "-lm"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout[-8000:])
        raise RuntimeError("building libref_raycast_emulated.so failed")


def build_marchingcubes_emulated():
    """The reference's iso-surface kernel (FL/DepthSensing/CUDAMarchingCubesSDF.cu with MarchingCubesSDFUtil.h, Tables.h, RayCastSDFUtil.h, VoxelUtilHashSDF.h,
    CUDAConstant.cu) compiled by g++ against the CUDA emulation -> libref_marchingcubes_emulated.so (wrapper: oracle/ref_marchingcubes_wrap.cu).  Runs on the CPU:
    pins row N4's marching-cubes oracle (and the triangle table) without a GPU.  Patches on the scratch copies: launch syntax, the HashEntry alignment attribute,
    the matNxM specialisation -- as for the ray cast."""
    root = os.path.join(TMP, "mcemu")
    os.makedirs(root)
    ds, sg = os.path.join(REF, "Source", "DepthSensing"), os.path.join(REF, "Source", "SiftGPU")
    for f in ("CUDAConstant.cu", "CUDAMarchingCubesSDF.cu", "MarchingCubesSDFUtil.h", "Tables.h", "RayCastSDFUtil.h", "VoxelUtilHashSDF.h", "DepthCameraUtil.h", "CUDAHashParams.h",
              "CUDADepthCameraParams.h", "CUDARayCastParams.h"):
        shutil.copy(os.path.join(ds, f), root)
    for f in ("cuda_SimpleMatrixUtil.h", "cudaUtil.h"):
        shutil.copy(os.path.join(sg, f), root)
    patch(os.path.join(root, "cuda_SimpleMatrixUtil.h"),
          [(r"\ninline __device__ __host__ matNxM<4, 1>::operator float4\(\)", "\ntemplate<> inline __device__ __host__ matNxM<4, 1>::operator float4()", 1)])
    for f in ("CUDAHashParams.h", "CUDADepthCameraParams.h", "CUDARayCastParams.h"):
        q = os.path.join(root, f)
        open(q, "w", encoding="latin-1").write("#pragma once\n" + open(os.path.join(ds, f), encoding="latin-1").read())
    patch(os.path.join(root, "VoxelUtilHashSDF.h"), [(r"__align__\(16\)\s*struct HashEntry", "struct __align__(16) HashEntry", 1)])
    patch(os.path.join(root, "RayCastSDFUtil.h"), [(r"float3 normal = -gradientForPoint\(hash, currentIso\);", "float3 g_ = gradientForPoint(hash, currentIso); float3 normal = -g_;", 1)])
    launch = (r"([A-Za-z_]\w*(?:<[^<>()]*>)?)\s*<<\s*<\s*([^;]*?)\s*>>\s*>\s*\(", r"EMU_KERNEL(\1, \2)(", None)
    patch(os.path.join(root, "CUDAMarchingCubesSDF.cu"), [launch])
    unit = os.path.join(root, "ref_marchingcubes_wrap_emu.cpp")
    shutil.copy(os.path.join(HERE, "ref_marchingcubes_wrap.cu"), unit)
    emu_dir = os.path.join(HERE, "ref_emu")
    cmd = ["g++", "-std=c++17", "-O2", "-w", "-fpermissive", "-ffp-contract=off", "-shared", "-fPIC", "-pthread", "-D__CUDACC__", "-D__NVCC__",
           "-I", emu_dir, "-I", os.path.join(os.path.dirname(HERE), "tests", "cuda_emu"), "-I", root, "-I", os.path.join(REF, "Include", "cutil", "inc"),
           unit, "-o", os.path.join(OUT, "libref_marchingcubes_emulated.so"), "-lm"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout[-8000:])
        raise RuntimeError("building libref_marchingcubes_emulated.so failed")


def prepare_mlib_scratch(root):
    """scratch copy of mLib's core headers (+ ext-depthcamera) with the seven one-line patches g++ needs (MSVC accepts the originals): a missing `typename`, calls of a
    member that does not exist inside never-instantiated templates (closeStream), a `w` in vec6::toString, unqualified dependent-base members in distanceField3.h, a
    typedef used before its declaration in material.h, `ios_base::open_mode`, `auto&` bound to a temporary in MeshData::isConsistent.  None touches the mesh clean-up,
    the PLY writer or the SensorData container.  Returns the g++ command prefix (C++17: mLib's face iterators declare a copy constructor from a non-const reference,
    which only guaranteed copy elision lets g++ accept) and the two mLib source files every user needs (warning / error hooks, util::)."""
    os.makedirs(root)
    mlib = os.path.join(os.path.dirname(REF), "external", "mLib", "include")
    for d in sorted(os.listdir(mlib)):
        if d.startswith("core-") or d == "ext-depthcamera":
            shutil.copytree(os.path.join(mlib, d), os.path.join(root, d))
    for f in ("mLibCore.h", "mLibDepthCamera.h"):
        shutil.copy(os.path.join(mlib, f), root)
    patch(os.path.join(root, "core-util", "binaryDataStream.h"), [(r"\n(\s*)BinaryDataBuffer::Mode mode = ", r"\n\1typename BinaryDataBuffer::Mode mode = ", 1), (r"in\.closeStream\(\);", "", None)])
    patch(os.path.join(root, "core-math", "vec6.h"), [(r"std::to_string\(z\) \+ separator \+ std::to_string\(w\) \+ separator \+", "std::to_string(z) + separator +", 1)])
    patch(os.path.join(root, "core-base", "distanceField3.h"), [(r"z < m_dimZ; z\+\+", "z < this->m_dimZ; z++", None), (r"y < m_dimY; y\+\+", "y < this->m_dimY; y++", None),
                                                                (r"x < m_dimX; x\+\+", "x < this->m_dimX; x++", None)])
    patch(os.path.join(root, "core-mesh", "material.h"), [(r"const Materialf& m0, const Materialf& m1", "const Material& m0, const Material& m1", 2)])
    patch(os.path.join(root, "core-util", "binaryDataBuffer.h"), [(r"std::ios_base::open_mode", "std::ios_base::openmode", None)])          # the pre-standard name, gone in C++17
    patch(os.path.join(root, "core-mesh", "meshData.h"), [(r"for \(auto& face : m_FaceIndices", "for (auto&& face : m_FaceIndices", 3)])    # isConsistent: reference to a temporary (MSVC extension)
    src = os.path.join(os.path.dirname(mlib), "src")
    return (["g++", "-std=c++17", "-O2", "-w", "-fpermissive", "-ffp-contract=off", "-shared", "-fPIC", "-DLINUX", "-I", root,
             "-include", "sys/types.h", "-include", "sys/stat.h", "-include", "unistd.h", "-include", "dirent.h", "-include", "mLibCore.h"],
            [os.path.join(src, "core-base", "common.cpp"), os.path.join(src, "core-util", "utility.cpp")])


def build_mesh_host():
    """The host half of the reference's mesh export: mLib's MeshDataf (mergeCloseVertices, removeDuplicateFaces, applyTransform) and MeshIOf::saveToFile, driven by
    the statements of CUDAMarchingCubesHashSDF::copyTrianglesToCPU / ::saveMesh (wrapper: oracle/ref_mesh_host.cpp) -> libref_mesh_host.so, g++ on mLib's headers
    where they lie (prepare_mlib_scratch)."""
    cmd, srcs = prepare_mlib_scratch(os.path.join(TMP, "meshhost"))
    r = subprocess.run(cmd + [os.path.join(HERE, "ref_mesh_host.cpp")] + srcs + ["-o", os.path.join(OUT, "libref_mesh_host.so")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout[-6000:])
        raise RuntimeError("building libref_mesh_host.so failed")


def build_sensordata_host():
    """The reference's `.sens` container class ml::SensorData (ext-depthcamera/sensorData.h; wrapper: oracle/ref_sensordata_host.cpp) -> libref_sensordata_host.so:
    writes files as the reference's recorder does (raw colour; JPEG / PNG compression is the Windows-only uplink codec) and reads files as its player does."""
    cmd, srcs = prepare_mlib_scratch(os.path.join(TMP, "sensdatahost"))
    stb = os.path.join(os.path.dirname(REF), "external", "mLib", "include", "mLibDepthCamera.cpp")                    # the stb_image / stb_image_write implementations (inside namespace stb)
    r = subprocess.run(cmd + ["-include", "assert.h", "-include", "stdarg.h", "-include", "limits.h", os.path.join(HERE, "ref_sensordata_host.cpp"), stb] + srcs +
                       ["-o", os.path.join(OUT, "libref_sensordata_host.so")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout[-6000:])
        raise RuntimeError("building libref_sensordata_host.so failed")


def build_sens_host():
    """The codecs behind the reference's `.sens` payloads: the stb_image / stb_image_write headers mLib vendors (external/mLib/include/ext-depthcamera/sensorData/),
    compiled by g++ where they lie -> libref_sens_host.so (wrapper: oracle/ref_sens_host.cpp).  Pins include/bf_sens.h's JPEG / PNG / zlib handling against the
    reference's decoder without a GPU."""
    ext = os.path.join(os.path.dirname(REF), "external", "mLib", "include", "ext-depthcamera")
    cmd = ["g++", "-std=c++17", "-O2", "-w", "-fpermissive", "-shared", "-fPIC", "-I", ext, os.path.join(HERE, "ref_sens_host.cpp"), "-o", os.path.join(OUT, "libref_sens_host.so")]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout[-6000:])
        raise RuntimeError("building libref_sens_host.so failed")


def build_trajectory_host():
    """The reference's TrajectoryManager (FL/TrajectoryManager.{h,cpp}) and the Lie part of FL/PoseHelper.h compiled by g++ against mLib's OWN math types
    (prepare_mlib_scratch) -> libref_trajectory_host.so (runs on the CPU).  oracle/ref_traj_stubs holds what is not mLib: stdafx.h (mLibCore.h, the POD float4x4 of the
    CUDA side, cudaMemcpy as memcpy), an empty CUDAImageManager.h and the two GlobalAppState settings the constructor reads.  (Until the g++ patches for mLib were
    found this was built against hand-written minimal vector / matrix types; the golden file that build produced is reproduced byte for byte by this one.)  Patch on the
    scratch copy of PoseHelper.h: the evaluation / file helpers in front of the pose maps are cut; the Lie pose maps are untouched.  Built -DNDEBUG like the reference's
    Release configuration (its asserts on list invariants fire on operation orders the application does not produce).  TrajectoryManager.cpp waits for a key press
    (getchar) after one of its error messages: drive the library with stdin closed."""
    root = os.path.join(TMP, "trajhost")
    cmd, srcs = prepare_mlib_scratch(os.path.join(TMP, "trajhost_mlib"))
    os.makedirs(root)
    S = os.path.join(REF, "Source")
    for f in ("TrajectoryManager.h", "TrajectoryManager.cpp", "PoseHelper.h", "GlobalDefines.h"):
        shutil.copy(os.path.join(S, f), root)
    patch(os.path.join(root, "PoseHelper.h"), [
        (r"\tstatic unsigned int countNumValidTransforms.*?(#ifndef USE_LIE_SPACE)", r"\1", 1),
    ])
    stubs = os.path.join(HERE, "ref_traj_stubs")
    r = subprocess.run(cmd + ["-DNDEBUG", "-I", stubs, "-I", root, os.path.join(HERE, "ref_trajectory_host.cpp"), os.path.join(root, "TrajectoryManager.cpp")] + srcs +
                       ["-o", os.path.join(OUT, "libref_trajectory_host.so"), "-lm"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout[-6000:])
        raise RuntimeError("building libref_trajectory_host.so failed")


if __name__ == "__main__":
    sys.exit(main())
