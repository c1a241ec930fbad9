"""Packaging for gllm_b200.

`pip install -e .` (or `pip install .`) compiles the sm_90a kernel library with nvcc through
`gllm_b200.build` — one shared object, no torch C++ headers — and ships it as package data.

Environment:
  GLLM_B200_SKIP_BUILD=1       do not run nvcc at install time (the library is then built on first import)
  GLLM_B200_PREBUILT_LIB=path  install this pre-built libgllm_b200.so instead of compiling (air-gapped
                               fleets that build once per image; the counterpart of the reference's
                               GLLM_PRECOMPILED_WHEEL_LOCATION, reference setup.py:198)
"""
import importlib.util
import os
import shutil

from setuptools import setup
from setuptools.command.build_py import build_py
from setuptools.command.develop import develop

HERE = os.path.dirname(os.path.abspath(__file__))


def _load_builder():
    # import gllm_b200/build.py by path: importing the package would pull torch in at install time
    spec = importlib.util.spec_from_file_location("_gllm_b200_build", os.path.join(HERE, "gllm_b200", "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def build_kernels():
    if os.environ.get("GLLM_B200_SKIP_BUILD") == "1":
        print("gllm_b200: GLLM_B200_SKIP_BUILD=1, kernel library will be built on first import")
        return
    b = _load_builder()
    prebuilt = os.environ.get("GLLM_B200_PREBUILT_LIB")
    if prebuilt:
        os.makedirs(b.OUT_DIR, exist_ok=True)
        shutil.copyfile(prebuilt, b.LIB_PATH)
        print(f"gllm_b200: installed pre-built kernel library {prebuilt}")
        return
    b.build(verbose=True)


class BuildPy(build_py):
    def run(self):
        build_kernels()
        super().run()


class Develop(develop):
    def run(self):
        build_kernels()
        super().run()


setup(cmdclass={"build_py": BuildPy, "develop": Develop})
