"""In-tree native build: nvcc (sm_90a) + g++ -> ``skycomputing_b200/_cuda*.so`` and ``_core*.so``.

The extensions are plain pybind11 modules (no libtorch linkage): ``_cuda`` holds every hand-written
sm_90a kernel, the CUDA-IPC peer-memory manager and the C++ device benchmark loop; ``_core`` holds
the C++ allocator / cost model / stimulator (no CUDA at all, importable on CPU-only boxes).

Build products stay in the package directory, so the package imports straight from the source
tree; a content-hash stamp next to them skips the rebuild when neither a source, a header nor a
flag changed.  ``python -m skycomputing_b200._build --force`` forces a build.
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
ROOT = PKG_DIR.parent
CSRC = ROOT / "csrc"
BUILD_DIR = ROOT / "build" / "obj"
EXT_SUFFIX = sysconfig.get_config_var("EXT_SUFFIX") or ".so"

CUDA_HOME = os.environ.get("CUDA_HOME", "/usr/local/cuda")
NVCC = os.path.join(CUDA_HOME, "bin", "nvcc")

CUDA_SOURCES = [
    "kernels/gemm_sm100.cu",
    "kernels/elementwise_sm100.cu",
    "kernels/attention_sm100.cu",
    "bench/device_bench.cu",
]
CUDA_BINDINGS = "bindings_cuda.cpp"
CORE_SOURCES = [
    "alloc/allocator.cc",
    "alloc/stimulator.cc",
    "bindings_core.cpp",
]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17", "--use_fast_math",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
]
CXX_FLAGS = ["-O2", "-std=c++17", "-fPIC", "-fvisibility=hidden", "-Wall"]


def _pybind_includes() -> list[str]:
    import pybind11

    return [f"-I{pybind11.get_include()}", f"-I{sysconfig.get_paths()['include']}"]


def _hash_files(files: list[Path], extra: str = "") -> str:
    h = hashlib.sha256()
    h.update(extra.encode())
    for f in sorted(files):
        h.update(str(f.relative_to(ROOT)).encode())
        h.update(f.read_bytes())
    return h.hexdigest()


def _run(cmd: list[str]) -> None:
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0:
        raise RuntimeError(
            "native build failed:\n$ " + " ".join(cmd) + "\n" + proc.stdout + proc.stderr
        )


def _headers() -> list[Path]:
    return sorted(list(CSRC.rglob("*.h")) + list(CSRC.rglob("*.cuh")) + list(CSRC.rglob("*.hpp")))


def so_path(name: str) -> Path:
    return PKG_DIR / f"{name}{EXT_SUFFIX}"


def _stamp_path(name: str) -> Path:
    return PKG_DIR / f".{name}.buildhash"


def _needs_build(name: str, digest: str) -> bool:
    so = so_path(name)
    st = _stamp_path(name)
    return not (so.exists() and st.exists() and st.read_text().strip() == digest)


def build_cuda(force: bool = False, verbose: bool = False) -> Path:
    srcs = [CSRC / s for s in CUDA_SOURCES] + [CSRC / CUDA_BINDINGS]
    digest = _hash_files(srcs + _headers(), extra=" ".join(NVCC_FLAGS))
    if not force and not _needs_build("_cuda", digest):
        return so_path("_cuda")
    if not os.path.exists(NVCC):
        raise RuntimeError(f"nvcc not found at {NVCC}; cannot build the sm_90a kernels")
    BUILD_DIR.mkdir(parents=True, exist_ok=True)
    objs: list[Path] = []
    jobs: list[list[str]] = []
    for s in CUDA_SOURCES:
        obj = BUILD_DIR / (s.replace("/", "_") + ".o")
        objs.append(obj)
        jobs.append([NVCC, *NVCC_FLAGS, f"-I{CSRC}", "-c", str(CSRC / s), "-o", str(obj)])
    bobj = BUILD_DIR / "bindings_cuda.o"
    objs.append(bobj)
    jobs.append(
        ["g++", *CXX_FLAGS, *_pybind_includes(), f"-I{CSRC}", f"-I{CUDA_HOME}/include", "-c",
         str(CSRC / CUDA_BINDINGS), "-o", str(bobj)]
    )
    if verbose:
        print(f"[skycomputing_b200] compiling {len(jobs)} native sources for sm_90a ...", flush=True)
    with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
        list(ex.map(_run, jobs))
    out = so_path("_cuda")
    tmp = out.with_suffix(out.suffix + ".tmp")
    _run(
        ["g++", "-shared", "-o", str(tmp), *map(str, objs), f"-L{CUDA_HOME}/lib64",
         "-lcudart_static", "-lrt", "-ldl", "-lpthread"]
    )
    os.replace(tmp, out)
    _stamp_path("_cuda").write_text(digest)
    return out


def build_core(force: bool = False, verbose: bool = False) -> Path:
    srcs = [CSRC / s for s in CORE_SOURCES]
    digest = _hash_files(srcs + _headers(), extra=" ".join(CXX_FLAGS))
    if not force and not _needs_build("_core", digest):
        return so_path("_core")
    BUILD_DIR.mkdir(parents=True, exist_ok=True)
    objs = []
    jobs = []
    for s in CORE_SOURCES:
        obj = BUILD_DIR / (s.replace("/", "_") + ".o")
        objs.append(obj)
        jobs.append(["g++", *CXX_FLAGS, *_pybind_includes(), f"-I{CSRC}", "-c", str(CSRC / s), "-o",
                     str(obj)])
    if verbose:
        print(f"[skycomputing_b200] compiling {len(jobs)} C++ core sources ...", flush=True)
    with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
        list(ex.map(_run, jobs))
    out = so_path("_core")
    tmp = out.with_suffix(out.suffix + ".tmp")
    _run(["g++", "-shared", "-o", str(tmp), *map(str, objs), "-lpthread"])
    os.replace(tmp, out)
    _stamp_path("_core").write_text(digest)
    return out


def build_all(force: bool = False, verbose: bool = True) -> None:
    build_core(force=force, verbose=verbose)
    build_cuda(force=force, verbose=verbose)


if __name__ == "__main__":
    build_all(force="--force" in sys.argv, verbose=True)
    print("built:", so_path("_core"), so_path("_cuda"))
