"""In-tree build of the native extensions (no pip, no JIT cache).

Two shared objects land next to this file so they travel with the source tree:

* ``_K``  - CUDA data-plane kernels for H100, ``nvcc -gencode arch=compute_90a,code=sm_90a``
            (sm_90a only; pybind11; no torch headers => seconds to build).
* ``_C``  - C++17 control plane (Lighthouse, ManagerServer, clients; pybind11).

Upstream torchft builds its native module with maturin/cargo
(pyproject.toml:1-3,39-44); our native code is C++/CUDA, so plain g++ and nvcc do.
"""

from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path
from typing import List

ROOT = Path(__file__).resolve().parent
CSRC = ROOT / "csrc"
BUILD = ROOT.parent / "build"
EXT = sysconfig.get_config_var("EXT_SUFFIX")

NVCC = os.environ.get("TFT_NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
# Use the system g++ (dynamic libstdc++, same one nvcc uses as host compiler and
# ABI-compatible with torch). $CXX may name a toolchain that links libstdc++
# STATICALLY -- two C++ runtimes in one process (ours + torch's) corrupt each
# other, so $CXX is deliberately ignored; override with TFT_CXX only.
CXX = os.environ.get("TFT_CXX") or ("/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++") or "g++")

GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]


def _includes() -> List[str]:
    import pybind11

    return [
        f"-I{pybind11.get_include()}",
        f"-I{sysconfig.get_paths()['include']}",
    ]


def _stamp(srcs: List[Path], flags: List[str]) -> str:
    h = hashlib.sha256()
    for s in sorted(srcs):
        h.update(s.name.encode())
        h.update(s.read_bytes())
    h.update(" ".join(flags).encode())
    return h.hexdigest()


def _run(cmd: List[str]) -> None:
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"build failed: {' '.join(cmd)}\n{r.stdout}\n{r.stderr}")
    if os.environ.get("TFT_BUILD_VERBOSE"):
        sys.stderr.write(r.stdout + r.stderr)


def build_kernels(force: bool = False, verbose: bool = False) -> Path:
    """Compile torchft_b200/_K*.so for sm_90a."""

    kdir = CSRC / "kernels"
    cus = sorted(kdir.glob("*.cu"))
    hdrs = sorted(kdir.glob("*.h")) + sorted(kdir.glob("*.cuh"))
    out = ROOT / f"_K{EXT}"
    flags = [
        "-O3",
        "-std=c++17",
        "-lineinfo",
        "--use_fast_math",
        "-Xcompiler",
        "-fPIC",
        "-Xcompiler",
        "-fvisibility=hidden",
        "--expt-relaxed-constexpr",
    ] + GENCODE
    if verbose or os.environ.get("TFT_PTXAS_V"):
        flags += ["-Xptxas", "-v"]
    stamp_file = BUILD / "_K.stamp"
    stamp = _stamp(cus + hdrs, flags)
    if not force and out.exists() and stamp_file.exists() and stamp_file.read_text() == stamp:
        return out
    odir = BUILD / "kernels"
    odir.mkdir(parents=True, exist_ok=True)
    objs = [odir / (c.stem + ".o") for c in cus]

    def cc(pair):
        src, obj = pair
        _run([NVCC, "-ccbin", CXX, "-c", str(src), "-o", str(obj)] + flags + _includes() + [f"-I{kdir}"])

    with ThreadPoolExecutor(max_workers=min(8, len(cus))) as ex:
        list(ex.map(cc, zip(cus, objs)))
    _run([NVCC, "-ccbin", CXX, "-shared", "-o", str(out)] + [str(o) for o in objs] + GENCODE + ["-cudart", "static"])
    stamp_file.write_text(stamp)
    return out


def build_control(force: bool = False) -> Path:
    """Compile torchft_b200/_C*.so (C++17 control plane)."""

    cdir = CSRC / "control"
    ccs = sorted(cdir.glob("*.cc"))
    hdrs = sorted(cdir.glob("*.h"))
    out = ROOT / f"_C{EXT}"
    flags = ["-O2", "-std=c++17", "-fPIC", "-fvisibility=hidden", "-pthread", "-Wall", "-Wno-unused-function"]
    stamp_file = BUILD / "_C.stamp"
    stamp = _stamp(ccs + hdrs, flags)
    if not force and out.exists() and stamp_file.exists() and stamp_file.read_text() == stamp:
        return out
    odir = BUILD / "control"
    odir.mkdir(parents=True, exist_ok=True)
    objs = [odir / (c.stem + ".o") for c in ccs]

    def cc(pair):
        src, obj = pair
        _run([CXX, "-c", str(src), "-o", str(obj)] + flags + _includes() + [f"-I{cdir}"])

    with ThreadPoolExecutor(max_workers=min(8, max(1, len(ccs)))) as ex:
        list(ex.map(cc, zip(ccs, objs)))
    _run([CXX, "-shared", "-o", str(out)] + [str(o) for o in objs] + ["-pthread"])
    stamp_file.write_text(stamp)
    return out


def build_lighthouse_binary(force: bool = False) -> Path:
    """Standalone `torchft_b200_lighthouse` executable (no Python needed)."""

    cdir = CSRC / "control"
    out = ROOT.parent / "bin" / "torchft_b200_lighthouse"
    srcs = [p for p in sorted(cdir.glob("*.cc")) if p.name != "bindings.cc"] + [cdir / "main" / "lighthouse_main.cpp"]
    srcs = [s for s in srcs if s.exists()]
    flags = ["-O2", "-std=c++17", "-pthread"]
    stamp_file = BUILD / "lighthouse_bin.stamp"
    stamp = _stamp(srcs + sorted(cdir.glob("*.h")), flags)
    if not force and out.exists() and stamp_file.exists() and stamp_file.read_text() == stamp:
        return out
    out.parent.mkdir(parents=True, exist_ok=True)
    BUILD.mkdir(parents=True, exist_ok=True)
    _run([CXX] + flags + [f"-I{cdir}"] + [str(s) for s in srcs] + ["-o", str(out)])
    stamp_file.write_text(stamp)
    return out


def build_selftest(force: bool = False, sanitize: str = "") -> Path:
    """Native unit/integration tests of the control plane (`cargo test` equivalent): bin/torchft_b200_selftest.

    ``sanitize="thread"`` / ``"address"`` builds the same tests under ThreadSanitizer / AddressSanitizer+UBSan
    (bin/torchft_b200_selftest_tsan / _asan) — the race and memory checks of the control plane."""

    cdir = CSRC / "control"
    suffix = {"": "", "thread": "_tsan", "address": "_asan"}[sanitize]
    out = ROOT.parent / "bin" / f"torchft_b200_selftest{suffix}"
    srcs = [cdir / f"{n}.cc" for n in ("wire", "quorum", "rpc", "lighthouse", "manager_server")] + [cdir / "tests" / "selftest.cc"]
    flags = ["-O1", "-g", "-std=c++17", "-pthread"]
    if sanitize == "thread":
        flags += ["-fsanitize=thread"]
    elif sanitize == "address":
        flags += ["-fsanitize=address,undefined", "-fno-omit-frame-pointer"]
    stamp_file = BUILD / f"selftest_bin{suffix}.stamp"
    stamp = _stamp(srcs + sorted(cdir.glob("*.h")), flags)
    if not force and out.exists() and stamp_file.exists() and stamp_file.read_text() == stamp:
        return out
    out.parent.mkdir(parents=True, exist_ok=True)
    BUILD.mkdir(parents=True, exist_ok=True)
    _run([CXX] + flags + [f"-I{cdir}"] + [str(s) for s in srcs] + ["-o", str(out)])
    stamp_file.write_text(stamp)
    return out


def build_all(force: bool = False, verbose: bool = False) -> None:
    BUILD.mkdir(parents=True, exist_ok=True)
    build_control(force=force)
    build_kernels(force=force, verbose=verbose)
    if (CSRC / "control" / "main" / "lighthouse_main.cpp").exists():
        build_lighthouse_binary(force=force)
    if (CSRC / "control" / "tests" / "selftest.cc").exists():
        build_selftest(force=force)


if __name__ == "__main__":
    build_all(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print("built:", sorted(p.name for p in ROOT.glob("_[CK]*.so")))
