"""``pip install --no-build-isolation -e .`` (or ``python setup.py build_ext --inplace``): builds the two C-ABI libraries in-tree
(``deeprec_b200/lib/libdeeprec_host.so`` with g++, ``libdeeprec_cuda.so`` with nvcc for sm_90a -- skipped with a warning when nvcc is
absent) through ``deeprec_b200/build.py`` and installs the python package around them."""
import os
import sys

from setuptools import Command, find_packages, setup
from setuptools.command.build_py import build_py

ROOT = os.path.dirname(os.path.abspath(__file__))


def _build_native():
    sys.path.insert(0, ROOT)
    import importlib.util
    spec = importlib.util.spec_from_file_location("deeprec_b200_build", os.path.join(ROOT, "deeprec_b200", "build.py"))
    b = importlib.util.module_from_spec(spec); spec.loader.exec_module(b)       # no `import deeprec_b200` (it would import torch)
    b.build_host()
    if os.path.exists(b.NVCC):
        b.build_cuda()
    else:
        print(f"warning: {b.NVCC} not found -- building the host library only (CPU training / serving)", file=sys.stderr)


class BuildNative(Command):
    description = "build libdeeprec_host.so / libdeeprec_cuda.so in-tree"
    user_options = [("inplace", "i", "accepted for build_ext compatibility (the build is always in-tree)")]

    def initialize_options(self):
        self.inplace = False

    def finalize_options(self):
        pass

    def run(self):
        _build_native()


class BuildPy(build_py):
    def run(self):
        _build_native()
        super().run()


setup(
    name="deeprec_b200",
    version="0.1.0",
    description="Hopper (H100) native sparse-recommender training and serving engine",
    packages=find_packages(include=["deeprec_b200", "deeprec_b200.*"]),
    package_data={"deeprec_b200": ["lib/*.so", "csrc/**/*", "csrc/*/*"]},
    python_requires=">=3.10",
    install_requires=["torch", "numpy"],
    extras_require={"serving": ["fastapi", "uvicorn", "prometheus_client", "grpcio"], "data": ["pyarrow", "pandas"]},
    cmdclass={"build_ext": BuildNative, "build_py": BuildPy},
    entry_points={"console_scripts": [
        "deeprec-train=deeprec_b200.models.train:main",
        "deeprec-serve=deeprec_b200.serving.serve:main",
        "deeprec-inspect-checkpoint=deeprec_b200.tools.inspect_checkpoint:main",
        "deeprec-ckpt-transform=deeprec_b200.tools.ckpt_format_transform:main",
    ]},
)
