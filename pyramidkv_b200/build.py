"""Build libpkv.so (sm_90a only) in-tree with nvcc. No JIT cache: the library is built once, next to the package."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libpkv.so")
SOURCES = ["pkv_api.cu", "pkv_score.cu", "pkv_score_tc5.cu", "pkv_topk.cu", "pkv_topk_cluster.cu", "pkv_gather.cu", "pkv_decode.cu", "pkv_h2o.cu", "pkv_l2norm.cu", "pkv_rope.cu", "pkv_flatten.cu", "pkv_h2o_tc5.cu", "pkv_adakv.cu", "pkv_evict_fused.cu", "pkv_fp8.cu", "pkv_install.cu", "pkv_sample.cu", "pkv_logprobs.cu", "pkv_rules.cu", "pkv_beam.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-Wall", "--expt-relaxed-constexpr", "-Xptxas", "-v",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found (needed to build pyramidkv_b200/libpkv.so for sm_90a)")


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "pkv.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    nvcc = _nvcc()
    env = dict(os.environ)
    # nvcc uses the system host compiler, whatever CC / CXX point at
    ccbin = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")
    procs = []
    for src in SOURCES:
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
        extra = ["-DPKV_STAMPS_BUILD"] if os.environ.get("PKV_BUILD_STAMPS") == "1" else []   # tools/stamps.py diagnostics
        cmd = [nvcc, "-ccbin", ccbin, *NVCC_FLAGS, *extra, "-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, obj, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env)))
    objs, log = [], []
    for src, obj, p in procs:
        out, _ = p.communicate()
        log.append(f"==== {src}\n{out}")
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}:\n{out}")
        objs.append(obj)
    link = [nvcc, "-ccbin", ccbin, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB, *objs]
    r = subprocess.run(link, capture_output=True, text=True, env=env)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}{r.stderr}")
    with open(os.path.join(objdir, "ptxas.log"), "w") as f:
        f.write("\n".join(log))
    if verbose:
        print("\n".join(log))
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
