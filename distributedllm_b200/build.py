"""Compile the sm_90a slice runtime in-tree: distributedllm_b200/libb200slice.so (+ the `llm` module).

nvcc cross-compiles without a GPU; the built .so files are git-ignored build products.
`python -m distributedllm_b200.build` or `build()`.
"""
from __future__ import annotations

import os
import subprocess
import sys
import sysconfig

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libb200slice.so")
LLM = os.path.join(HERE, "llm" + sysconfig.get_config_var("EXT_SUFFIX"))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
CU_SOURCES = ["runtime.cu"]          # one translation unit: kernels.cuh / fastgemm2.cuh are headers of it


def _newer(target: str, deps) -> bool:
    if not os.path.isfile(target):
        return False
    t = os.path.getmtime(target)
    return all(os.path.getmtime(d) <= t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    srcs = [os.path.join(CSRC, s) for s in CU_SOURCES if os.path.isfile(os.path.join(CSRC, s))]
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "b200_slice.h")]
    if force or not _newer(LIB, deps):
        objs = []
        procs = []
        os.makedirs(os.path.join(HERE, "..", "build"), exist_ok=True)
        for s in srcs:
            o = os.path.join(HERE, "..", "build", os.path.basename(s) + ".o")
            objs.append(o)
            cmd = [NVCC, *ARCH, "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC,-ffp-contract=off",
                   "-I/usr/include", "-c", s, "-o", o]
            cmd[1:1] = os.environ.get("B200_NVCC_DEFS", "").split()     # e.g. -DB200_TRACE_WAITS (main-loop wait counters)
            if verbose:
                cmd.insert(1, "-Xptxas=-v")
            procs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        for cmd, p in procs:
            out, _ = p.communicate()
            if verbose or p.returncode:
                sys.stderr.write(out)
            if p.returncode:
                raise RuntimeError("nvcc failed: " + " ".join(cmd))
        subprocess.run([NVCC, *ARCH, "-shared", "-o", LIB, *objs, "-ldl"], check=True)
    llm_src = os.path.join(CSRC, "llm_module.cpp")
    if os.path.isfile(llm_src) and (force or not _newer(LLM, [llm_src, LIB])):
        inc = sysconfig.get_paths()["include"]
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-I" + inc, "-I" + os.path.join(HERE, "..", "include"),
                        llm_src, "-o", LLM, "-L" + HERE, "-lb200slice", "-Wl,-rpath,$ORIGIN"], check=True)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
