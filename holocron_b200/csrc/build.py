"""Builds libholocron_b200.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a.

Usage: ``python -m holocron_b200.csrc.build [--force]``. Each ``.cu`` file is its own translation unit
(compiled in parallel), then linked with ``nvcc -shared``. The cudart runtime is linked statically so
that the library only depends on libcuda/libdl at load time; the TMA descriptor encoder
(``cuTensorMapEncode*``) is resolved at run time through ``cudaGetDriverEntryPoint`` so there is no
link-time dependency on libcuda either (the library builds on machines without a driver).
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

HERE = Path(__file__).resolve().parent
OBJ = HERE / "build"
LIB = HERE / "libholocron_b200.so"
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
CFLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
          "-Xptxas", "-v", "-I", str(HERE), "-I", str(HERE.parent.parent / "include")]


def _newer(src: Path, dst: Path, deps) -> bool:
    if not dst.exists():
        return True
    t = dst.stat().st_mtime
    return any(p.stat().st_mtime > t for p in [src, *deps])


def _compile(src: Path, force: bool) -> Path:
    obj = OBJ / (src.stem + ".o")
    deps = list(HERE.glob("*.cuh")) + list((HERE.parent.parent / "include").glob("*.h"))
    if force or _newer(src, obj, deps):
        cmd = [NVCC, *ARCH, *CFLAGS, "-c", str(src), "-o", str(obj)]
        res = subprocess.run(cmd, capture_output=True, text=True)
        log = OBJ / (src.stem + ".log")
        log.write_text(res.stdout + res.stderr)
        if res.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src.name}:\n{res.stdout}\n{res.stderr}")
    return obj


def build(force: bool = False, verbose: bool = False) -> Path:
    OBJ.mkdir(exist_ok=True)
    srcs = sorted(HERE.glob("*.cu"))
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(lambda s: _compile(s, force), srcs))
    if force or not LIB.exists() or any(o.stat().st_mtime > LIB.stat().st_mtime for o in objs):
        cmd = [NVCC, *ARCH, "-shared", "-cudart", "static", "-o", str(LIB), *map(str, objs), "-ldl"]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError(f"link failed:\n{res.stdout}\n{res.stderr}")
    if verbose:
        print(f"built {LIB} from {len(srcs)} translation units")
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose=True)
