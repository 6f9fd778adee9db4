"""Build hook: the native modules are compiled in-tree by ``torchft_b200/_build.py`` (nvcc for
sm_90a + g++ for the control plane) before setuptools collects the package, so an sdist/wheel or
``pip install -e .`` carries ``_K*.so`` / ``_C*.so`` and the lighthouse binary."""

import importlib.util
import os

from setuptools import setup
from setuptools.command.build_py import build_py


class BuildNative(build_py):
    def run(self):
        here = os.path.dirname(os.path.abspath(__file__))
        spec = importlib.util.spec_from_file_location("_tft_build", os.path.join(here, "torchft_b200", "_build.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        mod.build_all()
        super().run()


setup(cmdclass={"build_py": BuildNative})
