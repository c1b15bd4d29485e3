"""`python setup.py build_ext --inplace` (or `python -m ring_flash_attn_b200.build_ext`) builds the sm_90a
extension next to the sources; `pip install -e .` installs the package in development mode."""
from setuptools import find_packages, setup
from setuptools.command.build_ext import build_ext as _build_ext


class BuildSm100(_build_ext):
    def run(self):  # nvcc is driven directly (explicit -gencode arch=compute_90a,code=sm_90a)
        from ring_flash_attn_b200 import build_ext

        print(build_ext.build(verbose=True))


setup(packages=find_packages(include=["ring_flash_attn_b200", "ring_flash_attn_b200.*"]),
      cmdclass={"build_ext": BuildSm100}, package_data={"ring_flash_attn_b200": ["csrc/*", "_C*.so"]})
