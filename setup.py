"""In-tree build of the native module: ``python setup.py build_ext --inplace``.

Produces ``shallowspeed_b200/_C*.so`` for the H100 (sm_90a only); the .so is a build product and
stays out of git.

Link hygiene: some toolchains resolve ``-lstdc++`` to the static archive, which then collides with
the dynamic libstdc++ torch already loaded.  We name ``libstdc++.so.6`` and ``libnccl.so.2``
explicitly and verify DT_NEEDED after the build."""
import glob
import os
import subprocess
import sys

from setuptools import find_packages, setup
from torch.utils.cpp_extension import BuildExtension, CUDAExtension

ROOT = os.path.dirname(os.path.abspath(__file__))


def _nccl_root() -> str:
    import nvidia.nccl as _nccl  # namespace package: __file__ is None, __path__ is what exists

    for p in list(_nccl.__path__):
        if os.path.exists(os.path.join(p, "lib", "libnccl.so.2")) and os.path.exists(os.path.join(p, "include", "nccl.h")):
            return p
    raise RuntimeError("NCCL (nvidia.nccl wheel: lib/libnccl.so.2 + include/nccl.h) not found")


NCCL_ROOT = _nccl_root()
sources = (["csrc/bindings.cpp"] + sorted(glob.glob("csrc/kernels/*.cu")) + sorted(glob.glob("csrc/runtime/*.cpp"))
           + sorted(glob.glob("csrc/runtime/*.cu")))
include_dirs = [os.path.join(ROOT, "csrc"), os.path.join(NCCL_ROOT, "include")]
extra_link = [
    f"-L{os.path.join(NCCL_ROOT, 'lib')}", "-l:libnccl.so.2", f"-Wl,-rpath,{os.path.join(NCCL_ROOT, 'lib')}",
    "-l:libstdc++.so.6",
]

os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0a")
os.environ.setdefault("MAX_JOBS", str(os.cpu_count() or 4))


class CheckedBuild(BuildExtension):
    """BuildExtension + a DT_NEEDED check on what it produced."""

    def run(self):
        super().run()
        for ext in self.extensions:
            path = self.get_ext_fullpath(ext.name)
            dyn = subprocess.run(["readelf", "-d", path], capture_output=True, text=True, check=True).stdout
            for need in ("libstdc++.so.6", "libnccl.so.2"):
                if need not in dyn:
                    raise RuntimeError(f"{path}: {need} missing from DT_NEEDED (static libstdc++ / unlinked NCCL)")
            print(f"[setup.py] {os.path.basename(path)}: DT_NEEDED has libstdc++.so.6 and libnccl.so.2", file=sys.stderr)


setup(
    name="shallowspeed_b200",
    version="0.2.0",
    packages=find_packages(include=["shallowspeed_b200*"]),
    ext_modules=[
        CUDAExtension(
            name="shallowspeed_b200._C",
            sources=sources,
            include_dirs=include_dirs,
            extra_compile_args={
                "cxx": ["-O3", "-std=c++17"],
                "nvcc": ["-O3", "-std=c++17", "-lineinfo", "-gencode", "arch=compute_90a,code=sm_90a",
                         "--expt-relaxed-constexpr"],
            },
            extra_link_args=extra_link,
        )
    ],
    cmdclass={"build_ext": CheckedBuild.with_options(use_ninja=True)},
)
