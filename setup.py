"""Packaging for sparkflow_b200.  The native extensions are built IN-TREE by ``tools/build_ext.py`` (nvcc for sm_90a;
``sparkflow_b200/_C.so`` and ``_host.so`` sit next to the Python sources), so ``pip install -e .`` / ``python setup.py
develop`` only has to trigger that build and register the package."""
import os
import subprocess
import sys

from setuptools import Command, find_packages, setup
from setuptools.command.build_py import build_py

HERE = os.path.dirname(os.path.abspath(__file__))


def _build_native():
    subprocess.check_call([sys.executable, os.path.join(HERE, "tools", "build_ext.py")], cwd=HERE)


class BuildNative(Command):
    description = "compile the sm_90a CUDA kernels + C++ runtime into sparkflow_b200/_C.so and _host.so"
    user_options = []

    def initialize_options(self):
        pass

    def finalize_options(self):
        pass

    def run(self):
        _build_native()


class BuildPyWithNative(build_py):
    def run(self):
        if os.environ.get("SPARKFLOW_SKIP_NATIVE_BUILD") != "1":
            _build_native()
        super().run()


setup(
    name="sparkflow_b200",
    version="0.1.0",
    description="Hopper-native asynchronous parameter-server training with the sparkflow API",
    packages=find_packages(include=["sparkflow_b200", "sparkflow_b200.*"]),
    package_data={"sparkflow_b200": ["_C.so", "_host.so"]},
    python_requires=">=3.10",
    install_requires=["numpy", "torch"],
    cmdclass={"build_native": BuildNative, "build_py": BuildPyWithNative},
    zip_safe=False,
)
