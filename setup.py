"""Build script of torch_cgx_b200 (sm_90a only).

    python setup.py build_ext --inplace     # in-tree build: torch_cgx_b200/_C*.so
    pip install --no-build-isolation .       # regular install

Counterpart of the reference's setup.py (/root/reference/setup.py:1-93) minus
MPI/ROCm: the only native dependencies are the CUDA runtime and libtorch.
"""
import os
from pathlib import Path

from setuptools import find_packages, setup
from torch.utils.cpp_extension import BuildExtension, CUDAExtension

ROOT = Path(__file__).parent.resolve()
CSRC = Path("torch_cgx_b200") / "csrc"

SOURCES = [
    "common/plan.cc",
    "common/config.cc",
    "common/layers.cc",
    "common/sra_sim.cc",
    "comm/fd_channel.cc",
    "comm/loopback_communicator.cc",
    "comm/symmetric_heap.cc",
    "reduce/fused_sra.cc",
    "reduce/block_backend.cc",
    "reduce/reducers.cc",
    "pg/c10d_communicator.cc",
    "pg/comm_hook.cc",
    "engine/engine.cc",
    "kernels/sra_f32.cu",
    "kernels/sra_f16.cu",
    "kernels/sra_bf16.cu",
    "kernels/rs_f32.cu",
    "kernels/rs_f16.cu",
    "kernels/rs_bf16.cu",
    "kernels/ag_f32.cu",
    "kernels/ag_f16.cu",
    "kernels/ag_bf16.cu",
    "kernels/sra_dispatch.cu",
    "kernels/item_kernels.cu",
    "kernels/residual_relu.cu",
    "kernels/batchnorm_cl.cu",
    "kernels/quant_error.cu",
    "pg/process_group_cgx.cc",
    "bindings.cc",
]

# explicit -gencode: torch's own arch list is bypassed when one is present
NVCC_FLAGS = [
    "-O3",
    "-std=c++17",
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo",
    "--fmad=false",  # the CPU oracle must be bit-exact: FMAs are written explicitly (quant_math.h)
    "-Xptxas", "-v",
]
CXX_FLAGS = ["-O3", "-std=c++17", "-ffp-contract=off", "-Wno-unused-function"]
# This image's default compiler wrapper (/opt/gcc/bin/g++) finds only a *static*
# libstdc++ (its libstdc++.so symlink dangles); a private static copy inside a
# Python extension has uninitialised locale state and segfaults on the first
# ostream insertion. Always link the system's shared libstdc++ explicitly.
LINK_FLAGS = []
for _d in ("/usr/lib/x86_64-linux-gnu", "/lib/x86_64-linux-gnu"):
    if (Path(_d) / "libstdc++.so.6").exists():
        LINK_FLAGS = [f"-L{_d}", "-l:libstdc++.so.6"]
        break

LINK_FLAGS.append("-ldl")  # nvtx3 (header-only) resolves the tool's injection library with dlopen

os.environ.setdefault("MAX_JOBS", str(os.cpu_count() or 4))

setup(
    name="torch_cgx_b200",
    version="0.1.0",
    description="Hopper-native compressed-gradient allreduce backend for torch.distributed",
    packages=find_packages(include=["torch_cgx_b200*", "torch_cgx", "cgx_utils"]),
    ext_modules=[
        CUDAExtension(
            name="torch_cgx_b200._C",
            sources=[str(CSRC / s) for s in SOURCES],
            extra_compile_args={"cxx": CXX_FLAGS, "nvcc": NVCC_FLAGS},
            extra_link_args=LINK_FLAGS,
        )
    ],
    cmdclass={"build_ext": BuildExtension.with_options(use_ninja=True, no_python_abi_suffix=False)},
    python_requires=">=3.10",
)
