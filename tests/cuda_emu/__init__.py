"""TEST INFRASTRUCTURE ONLY: builds a CPU-executable twin of a csrc/ source on top of cuda_emu.h (see its header), and runs the library's
host-side refusals in a process that sees no CUDA device."""
import ctypes as C
import functools
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
CSRC = os.path.join(ROOT, "bundlefusion_b200", "csrc")
EMU = os.path.join(ROOT, "tests", "cuda_emu")


@functools.lru_cache(maxsize=None)
def build_emulated(source: str, expected_launches: int, extra_pre: str = "", glue: str = "", sequential: bool = False) -> C.CDLL:
    """compile csrc/`source` (a .cu file, or a device header the `glue` launches from) for the CPU and load it.  `extra_pre` goes before the
    source, `glue` (the test's extern "C" wrappers) after it.  The source's <<<...>>> launches become EMU_LAUNCH, `expected_launches` of them.
    `sequential` runs each launch one CUDA thread after the other (BF_EMU_SEQUENTIAL, for sources that drop their warp collectives under it).
    One build per set of arguments and session."""
    src = open(os.path.join(CSRC, source)).read()
    # the library's own device headers are spliced in (they include bf_common.cuh, which the shim replaces)
    src = re.sub(r'#include "(\w+\.cuh)"', lambda m: m.group(0) if m.group(1) == "bf_common.cuh" else open(os.path.join(CSRC, m.group(1))).read(), src)
    src = src.replace('#include "bf_common.cuh"', "").replace("#pragma once", "")
    src = re.sub(r"extern __shared__ float (\w+)\[\];", lambda m: "" if m.group(1) == "sm" else f"float* {m.group(1)} = sm;", src)      # dynamic shared memory: the shim's sm[]
    src = re.sub(r"extern __shared__ (unsigned|int) (\w+)\[\];", lambda m: f"{m.group(1)}* {m.group(2)} = reinterpret_cast<{m.group(1)}*>(sm);", src)
    src, n = re.subn(r"(\w+(?:<[\w\s,]+>)?)<<<\s*([^,]+),\s*([^,]+),\s*[^,]+,\s*[^>]+>>>\(", r"EMU_LAUNCH((\1), \2, \3, ", src)
    assert n == expected_launches, (source, n)
    pre = ("#define BF_EMU_SEQUENTIAL 1\n" if sequential else "") + '#include "%s"\n' % os.path.join(EMU, "cuda_emu.h") + (
        "#define BF_CHECK(e) do { int _e = (int)(e); if (_e) return _e; } while (0)\n#define BF_SAFE(e) do { (void)(e); } while (0)\n"
        "namespace bf { unsigned long long g_launchCount = 0; static inline cudaStream_t stream() { return nullptr; } static inline int num_sms() { return 2; } }\n")
    if sequential:
        pre += "static inline unsigned warp_sum_u(unsigned v) { return v; }      // a warp of one thread\n"
    d = tempfile.mkdtemp(prefix="bf_emu_")
    try:
        stem = os.path.splitext(source)[0] + "_emu"
        cpp, so = os.path.join(d, stem + ".cpp"), os.path.join(d, "lib" + stem + ".so")
        open(cpp, "w").write(pre + extra_pre + src + glue)
        r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-pthread", "-I", EMU, "-I", CSRC, cpp, "-o", so],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-4000:]
        return C.CDLL(so)
    finally:
        shutil.rmtree(d, ignore_errors=True)           # the mapping outlives the file


def run_without_device(script: str) -> dict:
    """run `script` (argv[1]: the repository root) in a child process that sees no CUDA device, so a library call that got past its host-side
    checks would fail in the CUDA runtime instead of touching memory; returns the JSON object the script prints last"""
    r = subprocess.run([sys.executable, "-c", script, ROOT], capture_output=True, text=True, env=dict(os.environ, CUDA_VISIBLE_DEVICES=""), cwd=ROOT,
                       timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])
