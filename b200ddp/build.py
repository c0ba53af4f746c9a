"""In-tree build of the sm_90a (H100) extension ``b200ddp/_C*.so``.

Explicit nvcc / g++ invocations (no JIT cache under ~/.cache: the built ``.so`` sits in the package
directory, where ``_ext`` imports it from).  ``-gencode arch=compute_90a,code=sm_90a`` is passed
directly, which bypasses torch's own arch list (the wgmma / TMA kernels need the ``a`` target);
``-lineinfo`` keeps profiler source views usable.  Objects are rebuilt only when the content hash of
(source + headers + flags) changes.
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

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
BUILD = PKG / "_build"
EXT_NAME = "_C"

CUDA_SOURCES = ["allreduce.cu", "broadcast.cu", "optim.cu", "loss.cu", "layernorm.cu", "linear_small.cu", "input.cu",
                "gemm_wgmma.cu", "batchnorm.cu", "pool.cu", "conv_wgmma.cu", "conv_wgrad_wgmma.cu", "conv_stem.cu", "fp8.cu",
                "attention.cu", "rotary.cu"]
CPP_SOURCES = ["peer_mem.cpp", "reducer.cpp", "bindings.cpp"]

ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]


def ext_path() -> Path:
    return PKG / (EXT_NAME + sysconfig.get_config_var("EXT_SUFFIX"))


def _cuda_home() -> str:
    for cand in (os.environ.get("CUDA_HOME"), os.environ.get("CUDA_PATH"), "/usr/local/cuda"):
        if cand and os.path.exists(os.path.join(cand, "bin", "nvcc")):
            return cand
    nvcc = shutil.which("nvcc")
    if nvcc:
        return str(Path(nvcc).resolve().parent.parent)
    raise RuntimeError("nvcc not found; set CUDA_HOME")


def _flags():
    import torch
    from torch.utils import cpp_extension as ce
    cuda_home = _cuda_home()
    includes = [str(CSRC)] + ce.include_paths("cuda") + [os.path.join(cuda_home, "include"), sysconfig.get_paths()["include"]]
    inc = []
    for p in dict.fromkeys(includes):
        inc += ["-isystem" if "site-packages" in p or "cuda" in p else "-I", p]
    abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
    common = [f"-D_GLIBCXX_USE_CXX11_ABI={abi}", f"-DTORCH_EXTENSION_NAME={EXT_NAME}", "-DTORCH_API_INCLUDE_EXTENSION_H",
              "-DPYBIND11_COMPILER_TYPE=\"_gcc\"", "-DPYBIND11_STDLIB=\"_libstdcpp\"", "-DPYBIND11_BUILD_ABI=\"_cxxabi1018\""]
    # pybind ABI tags must match torch's so at::Tensor casters interoperate
    try:
        common = [f"-D_GLIBCXX_USE_CXX11_ABI={abi}", f"-DTORCH_EXTENSION_NAME={EXT_NAME}", "-DTORCH_API_INCLUDE_EXTENSION_H"]
        for name in ("COMPILER_TYPE", "STDLIB", "BUILD_ABI"):
            val = getattr(torch._C, f"_PYBIND11_{name}", None)
            if val is not None:
                common.append(f'-DPYBIND11_{name}="{val}"')
    except Exception:
        pass
    nvcc = [os.path.join(cuda_home, "bin", "nvcc"), *ARCH_FLAGS, "-lineinfo", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
            "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "-diag-suppress", "177", *common, *inc]
    cxx = [os.environ.get("CXX", "g++"), "-O2", "-std=c++17", "-fPIC", "-fvisibility=hidden", "-Wno-unused-variable", *common, *inc]
    torch_lib = os.path.join(os.path.dirname(torch.__file__), "lib")
    link = [os.environ.get("CXX", "g++"), "-shared", "-o", str(ext_path())]
    libs = ["-L" + torch_lib, "-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda", "-ltorch", "-ltorch_python",
            "-L" + os.path.join(cuda_home, "lib64"), "-lcudart", "-ldl", "-Wl,-rpath," + torch_lib, "-Wl,--no-as-needed"]
    return nvcc, cxx, link, libs


def _digest(src: Path, cmd) -> str:
    h = hashlib.sha256()
    h.update(" ".join(cmd).encode())
    h.update(src.read_bytes())
    for hdr in sorted(list(CSRC.glob("*.h")) + list(CSRC.glob("*.cuh"))):
        h.update(hdr.name.encode())
        h.update(hdr.read_bytes())
    return h.hexdigest()


def _compile(src_name: str, base_cmd, verbose: bool) -> tuple[Path, bool]:
    src = CSRC / src_name
    obj = BUILD / (src_name + ".o")
    stamp = BUILD / (src_name + ".sha")
    cmd = [*base_cmd, "-c", str(src), "-o", str(obj)]
    digest = _digest(src, base_cmd)
    if obj.exists() and stamp.exists() and stamp.read_text() == digest:
        return obj, False
    if verbose:
        print(f"[b200ddp.build] compiling {src_name}", flush=True)
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0:
        raise RuntimeError(f"compiling {src_name} failed:\n{proc.stdout}\n{proc.stderr}")
    stamp.write_text(digest)
    return obj, True


def build(verbose: bool = True, force: bool = False) -> Path:
    BUILD.mkdir(exist_ok=True)
    if force:
        for f in BUILD.glob("*.sha"):
            f.unlink()
    nvcc, cxx, link, libs = _flags()
    jobs = [(s, nvcc) for s in CUDA_SOURCES] + [(s, cxx) for s in CPP_SOURCES]
    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 4)) as pool:
        results = list(pool.map(lambda j: _compile(j[0], j[1], verbose), jobs))
    objs = [str(o) for o, _ in results]
    changed = any(c for _, c in results)
    out = ext_path()
    if changed or not out.exists():
        if verbose:
            print(f"[b200ddp.build] linking {out.name}", flush=True)
        proc = subprocess.run([*link, *objs, *libs], capture_output=True, text=True)
        if proc.returncode != 0:
            raise RuntimeError(f"linking failed:\n{proc.stdout}\n{proc.stderr}")
    return out


if __name__ == "__main__":
    path = build(verbose=True, force="--force" in sys.argv)
    print(path)
