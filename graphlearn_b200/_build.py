"""In-tree build of the native extension ``graphlearn_b200._C``.

Compiles every ``csrc/*.cu`` / ``*.cpp`` for sm_90a only
(``-gencode arch=compute_90a,code=sm_90a -lineinfo``) with
``torch.utils.cpp_extension`` and leaves the resulting ``_C.so`` inside the
package directory, so that the snapshot shipped to a GPU box already contains
the binary (a JIT cache under ~/.cache would not travel).
"""
from __future__ import annotations

import glob
import hashlib
import importlib
import importlib.util
import os
import shutil
import sys

_PKG_DIR = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(_PKG_DIR, "csrc")
_INCLUDE = os.path.join(_PKG_DIR, "include")      # public C++ headers (include/glb/api.h)
_BUILD_DIR = os.path.join(_PKG_DIR, "build")
_SO_PATH = os.path.join(_PKG_DIR, "_C.so")
_STAMP = os.path.join(_PKG_DIR, "_C.stamp")

CUDA_FLAGS = [
    "-O3",
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo",
    "--expt-relaxed-constexpr",
    "-Xptxas", "-v",
    "-U__CUDA_NO_HALF_OPERATORS__", "-U__CUDA_NO_HALF_CONVERSIONS__",
    "-U__CUDA_NO_BFLOAT16_CONVERSIONS__", "-U__CUDA_NO_HALF2_OPERATORS__",
]
CXX_FLAGS = ["-O3", "-std=c++17", "-fPIC"]


def sources():
    srcs = sorted(glob.glob(os.path.join(_CSRC, "*.cu")) + glob.glob(os.path.join(_CSRC, "*.cpp")))
    return srcs


def _digest():
    h = hashlib.sha256()
    for f in sorted(glob.glob(os.path.join(_CSRC, "*")) + glob.glob(os.path.join(_INCLUDE, "glb", "*"))):
        if os.path.isfile(f):
            h.update(f.encode())
            with open(f, "rb") as fh:
                h.update(fh.read())
    h.update(" ".join(CUDA_FLAGS + CXX_FLAGS).encode())
    return h.hexdigest()


def is_fresh() -> bool:
    if not (os.path.exists(_SO_PATH) and os.path.exists(_STAMP)):
        return False
    with open(_STAMP) as fh:
        return fh.read().strip() == _digest()


def build(verbose: bool = False, force: bool = False) -> str:
    """Build (if stale) and return the path of the in-tree shared object."""
    if is_fresh() and not force:
        return _SO_PATH
    # torch's own arch list must not add more -gencode flags
    os.environ["TORCH_CUDA_ARCH_LIST"] = "9.0a"
    os.environ.setdefault("MAX_JOBS", str(max(1, (os.cpu_count() or 4) - 1)))
    from torch.utils import cpp_extension

    os.makedirs(_BUILD_DIR, exist_ok=True)
    cpp_extension.load(
        name="_C",
        sources=sources(),
        extra_cflags=CXX_FLAGS,
        extra_cuda_cflags=CUDA_FLAGS,
        extra_include_paths=[_CSRC, _INCLUDE],
        build_directory=_BUILD_DIR,
        with_cuda=True,
        is_python_module=False,   # just build; we import from the in-tree copy below
        verbose=verbose,
    )
    built = os.path.join(_BUILD_DIR, "_C.so")
    if not os.path.exists(built):
        raise RuntimeError("extension build produced no _C.so")
    shutil.copy2(built, _SO_PATH)
    with open(_STAMP, "w") as fh:
        fh.write(_digest())
    return _SO_PATH


def load(build_if_missing: bool = True):
    """Import ``graphlearn_b200._C`` from the in-tree .so."""
    name = "graphlearn_b200._C"
    if name in sys.modules:
        return sys.modules[name]
    if not os.path.exists(_SO_PATH):
        if not build_if_missing:
            raise ImportError("graphlearn_b200/_C.so is missing; run `python -m graphlearn_b200._build`")
        build()
    import torch  # noqa: F401  (libtorch symbols must be loaded first)

    spec = importlib.util.spec_from_file_location(name, _SO_PATH)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    sys.modules[name] = mod
    return mod


if __name__ == "__main__":
    p = build(verbose=True, force="--force" in sys.argv)
    print("built", p)
