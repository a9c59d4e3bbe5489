"""Build the reference's path_creator.pyx into oracle/_ref/path_creator/ (TEST INFRASTRUCTURE ONLY).

Compiles the reference's src/urh/cythonext/path_creator.pyx (in the tree oracle/build_ref.py reads), unmodified and where it
lies, with the directives and flags oracle/build_ref.py uses for the other Cython modules.  It lives in its own directory so that oracle/ref_loader.py, which puts an
empty stand-in module in place of urh.cythonext.path_creator, sees no change.  The module imports PyQt6 at import time; the tests
load it with ``load()`` on top of ref_loader's Qt stub and swap a Qt fake in for the duration of a call.

Usage:  python oracle/build_ref_path_creator.py   (no-op where the reference tree is absent)
"""
import importlib.machinery
import importlib.util
import os
import shutil
import sys
import sysconfig

HERE = os.path.dirname(os.path.abspath(__file__))
if os.path.dirname(HERE) not in sys.path:
    sys.path.insert(0, os.path.dirname(HERE))
from oracle.build_ref import REF, ref_available  # noqa: E402

OUT = os.path.join(HERE, "_ref", "path_creator")
SO = os.path.join(OUT, "urh", "cythonext", "path_creator" + sysconfig.get_config_var("EXT_SUFFIX"))


def built() -> bool:
    return os.path.isfile(SO)


def build(force: bool = False) -> bool:
    if not os.path.isfile(os.path.join(REF, "src/urh/cythonext/path_creator.pyx")) or not ref_available():
        return built()
    if built() and not force:
        return True
    os.environ["CC"] = "/usr/bin/gcc"   # as oracle/build_ref.py: the default wrapper cannot link -fopenmp
    os.environ["CXX"] = "/usr/bin/g++"
    os.environ["LDSHARED"] = "/usr/bin/g++ -shared"
    import numpy as np
    from Cython.Build import cythonize
    from setuptools import Extension
    from setuptools.command.build_ext import build_ext
    from setuptools.dist import Distribution

    src_dir = os.path.join(REF, "src")
    ext = Extension(
        "urh.cythonext.path_creator",
        [os.path.join(src_dir, "urh", "cythonext", "path_creator.pyx")],
        extra_compile_args=["-fopenmp", "-O2", "-Wno-cpp", "-w"],
        extra_link_args=["-fopenmp"],
        include_dirs=[np.get_include()],
        language="c++",
    )
    cwd = os.getcwd()
    os.chdir(src_dir)   # so that the urh.cythonext.util cimport resolves; nothing is written here
    try:
        exts = cythonize(
            [ext],
            build_dir=os.path.join(OUT, "_gen"),
            include_path=[src_dir],
            compiler_directives=dict(language_level=3, cdivision=True, wraparound=False, boundscheck=False, initializedcheck=False),
            quiet=True,
        )
        cmd = build_ext(Distribution({"ext_modules": exts}))
        cmd.build_lib = OUT
        cmd.build_temp = os.path.join(OUT, "_tmp")
        cmd.inplace = 0
        cmd.ensure_finalized()
        cmd.run()
    finally:
        os.chdir(cwd)
    shutil.rmtree(os.path.join(OUT, "_tmp"), ignore_errors=True)
    shutil.rmtree(os.path.join(OUT, "_gen"), ignore_errors=True)
    return built()


_module = None


def load():
    """the compiled reference module (needs the reference's Python layer for `from urh import settings`); not registered in
    sys.modules, so ref_loader's stand-in for urh.cythonext.path_creator stays where it is"""
    global _module
    if _module is None:
        from oracle import ref_loader

        ref_loader.load_kernels()   # Qt stub, the reference's urh package
        if not built():
            raise ImportError("oracle/_ref/path_creator not built (run python oracle/build_ref_path_creator.py)")
        import urh.settings  # noqa: F401
        loader = importlib.machinery.ExtensionFileLoader("urh.cythonext.path_creator", SO)
        spec = importlib.util.spec_from_file_location("urh.cythonext.path_creator", SO, loader=loader)
        mod = importlib.util.module_from_spec(spec)
        loader.exec_module(mod)
        _module = mod
    return _module


if __name__ == "__main__":
    ok = build(force="--force" in sys.argv)
    print("oracle/_ref/path_creator built:", ok)
    sys.exit(0 if ok or not ref_available() else 1)
