"""In-tree build of the sm_90a (H100) extension (``lstm_tensorspark_b200/_C*.so``).

Kernels (``csrc/*.cu``) are compiled by plain ``nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo`` —
they depend on the CUDA runtime only, so a file builds in seconds and ``cuobjdump -sass`` of the result is
readable; ``csrc/bindings.cpp`` (the only translation unit that sees torch headers) is compiled by g++ and
everything is linked into ONE shared object next to the package so it travels with the source tree.
nvcc cross-compiles without a GPU, so this runs on a machine without one.

    python -m lstm_tensorspark_b200.build [--force] [--verbose] [--sass]
"""
from __future__ import annotations

import concurrent.futures as cf
import hashlib
import json
import os
import shutil
import subprocess
import sys
import sysconfig
from typing import List

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
BUILD = os.path.join(HERE, "build")
SO_NAME = "_C" + (sysconfig.get_config_var("EXT_SUFFIX") or ".so")
SO_PATH = os.path.join(HERE, SO_NAME)

ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ["-O3", "-std=c++17", "-lineinfo", "--use_fast_math", "-Xcompiler", "-fPIC", "-Xptxas", "-v",
              "--expt-relaxed-constexpr", "-DNDEBUG"] + ARCH_FLAGS


def _nvcc() -> str:
    cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    return cand if os.path.exists(cand) else (shutil.which("nvcc") or "nvcc")


def _cuda_home() -> str:
    return os.environ.get("CUDA_HOME", "/usr/local/cuda")


def _hash(paths: List[str], extra: str) -> str:
    h = hashlib.sha256(extra.encode())
    for p in sorted(paths):
        with open(p, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def _run(cmd: List[str], log_path: str, verbose: bool) -> None:
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    with open(log_path, "w") as f:
        f.write(" ".join(cmd) + "\n" + r.stdout)
    if verbose or r.returncode != 0:
        sys.stderr.write(r.stdout)
    if r.returncode != 0:
        raise RuntimeError(f"build step failed ({r.returncode}): {' '.join(cmd)}\n{r.stdout[-4000:]}")


def sources():
    cus = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))
    hdrs = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h")))
    cpp = os.path.join(CSRC, "bindings.cpp")
    return cus, hdrs, cpp


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(BUILD, exist_ok=True)
    cus, hdrs, cpp = sources()
    stamp_path = os.path.join(BUILD, "stamps.json")
    stamps = {}
    if os.path.isfile(stamp_path) and not force:
        try:
            stamps = json.load(open(stamp_path))
        except Exception:
            stamps = {}
    hdr_hash = _hash(hdrs, "hdr")
    jobs = []
    objs = []
    for cu in cus:
        obj = os.path.join(BUILD, os.path.basename(cu)[:-3] + ".o")
        objs.append(obj)
        key = _hash([cu], hdr_hash + " ".join(NVCC_FLAGS))
        if stamps.get(cu) == key and os.path.isfile(obj):
            continue
        cmd = [_nvcc()] + NVCC_FLAGS + ["-I", CSRC, "-c", cu, "-o", obj]
        jobs.append((cu, key, cmd, obj + ".log"))

    import torch
    from torch.utils import cpp_extension as ce
    inc = []
    for p in ce.include_paths():
        inc += ["-isystem", p]
    inc += ["-isystem", sysconfig.get_paths()["include"], "-isystem", os.path.join(_cuda_home(), "include")]
    cpp_obj = os.path.join(BUILD, "bindings.o")
    abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
    cxx_flags = ["-O2", "-std=c++17", "-fPIC", "-DTORCH_EXTENSION_NAME=_C", "-DTORCH_API_INCLUDE_EXTENSION_H",
                 f"-D_GLIBCXX_USE_CXX11_ABI={abi}", "-Wno-deprecated-declarations"]
    cpp_key = _hash([cpp], hdr_hash + " ".join(cxx_flags) + torch.__version__)
    if stamps.get(cpp) != cpp_key or not os.path.isfile(cpp_obj):
        jobs.append((cpp, cpp_key, ["g++"] + cxx_flags + inc + ["-c", cpp, "-o", cpp_obj], cpp_obj + ".log"))

    if jobs:
        with cf.ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            futs = {ex.submit(_run, cmd, log, verbose): (src, key) for (src, key, cmd, log) in jobs}
            for fut in cf.as_completed(futs):
                src, key = futs[fut]
                fut.result()
                stamps[src] = key
        json.dump(stamps, open(stamp_path, "w"), indent=1)

    need_link = bool(jobs) or not os.path.isfile(SO_PATH)
    if need_link:
        torch_lib = os.path.join(os.path.dirname(torch.__file__), "lib")
        link = ["g++", "-shared", "-o", SO_PATH, cpp_obj] + objs + [
            f"-L{torch_lib}", "-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda", "-ltorch", "-ltorch_python",
            f"-L{os.path.join(_cuda_home(), 'lib64')}", "-lcudart",
            f"-Wl,-rpath,{torch_lib}", f"-Wl,-rpath,{os.path.join(_cuda_home(), 'lib64')}"]
        _run(link, os.path.join(BUILD, "link.log"), verbose)
    return SO_PATH


def dump_sass(out_dir: str) -> List[str]:
    """``cuobjdump -sass`` per kernel object -> docs/sass/<name>.sass (committed evidence)."""
    os.makedirs(out_dir, exist_ok=True)
    outs = []
    cus, _, _ = sources()
    for cu in cus:
        obj = os.path.join(BUILD, os.path.basename(cu)[:-3] + ".o")
        if not os.path.isfile(obj):
            continue
        r = subprocess.run([os.path.join(_cuda_home(), "bin", "cuobjdump"), "-sass", obj], stdout=subprocess.PIPE,
                           stderr=subprocess.STDOUT, text=True)
        p = os.path.join(out_dir, os.path.basename(cu)[:-3] + ".sass")
        text = r.stdout
        keep = SASS_KEEP.get(os.path.basename(cu))
        if keep:
            text = _filter_sass(text, keep)
        with open(p, "w") as f:
            f.write(text)
        outs.append(p)
    return outs


# lstm_seq_wgmma.cu has ~120 template instantiations (ring depths, tuning variants, each with and without per-row lengths, in both
# time directions): the listing keeps the unmasked forward-time forward and backward kernels with one and two batch tiles per CTA
# at the ring depths H = 1024 gets, the streamed-weights kernels and the prologue.
# gemm2_wgmma.cu has 48 (cluster size x tile x operand majors x output mode); kept: the default 2-CTA 256-wide kernels of the
# x-projection (TN, bf16 out), dX (B MN-major, bf16 out) and the weight gradients (both MN-major, fp32 accumulate).
SASS_KEEP = {"lstm_seq_wgmma.cu": ("ILb0ELi4ELi1ELb0ELb0ELb0ELb0E", "ILb0ELi4ELi2ELb0ELb0ELb0ELb0E", "ILb1ELi3ELi1ELb0ELb0ELb0ELb0E",
                                  "ILb1ELi2ELi2ELb0ELb0ELb0ELb0E", "ILb0ELi8ELi1ELb1ELb0ELb0ELb0E", "ILb1ELi8ELi1ELb1ELb0ELb0ELb0E",
                                  "seq_prologue_kernel"),
             "gemm2_wgmma.cu": ("ILi2ELi256ELb0ELb0ELi0E", "ILi2ELi256ELb0ELb1ELi0E", "ILi2ELi256ELb1ELb1ELi2E")}


def _filter_sass(text: str, keep) -> str:
    parts = text.split("\t\tFunction : ")
    out = [parts[0]]
    for part in parts[1:]:
        name = part.split("\n", 1)[0]
        if any(k in name for k in keep):
            out.append(part)
    return "\t\tFunction : ".join(out)


def ptxas_report() -> str:
    """Registers / spills / smem per kernel, collected from the nvcc logs."""
    lines = []
    for f in sorted(os.listdir(BUILD)):
        if f.endswith(".o.log"):
            txt = open(os.path.join(BUILD, f)).read().splitlines()
            for i, l in enumerate(txt):
                if "Compiling entry function" in l or "Used " in l or "spill" in l:
                    lines.append(f"{f[:-6]}: {l.strip()}")
    return "\n".join(lines)


if __name__ == "__main__":
    force = "--force" in sys.argv
    verbose = "--verbose" in sys.argv
    path = build(force=force, verbose=verbose)
    print("built", path)
    if "--sass" in sys.argv:
        root = os.path.dirname(HERE)
        print("\n".join(dump_sass(os.path.join(root, "docs", "sass"))))
    if "--report" in sys.argv:
        print(ptxas_report())
