"""Build the reference's own Cython DSP kernels into oracle/_ref/ (TEST INFRASTRUCTURE ONLY).

Compiles, unmodified and where they lie, the three hot-path .pyx files of the reference
(/root/reference/src/urh/cythonext/{signal_functions,util,auto_interpretation}.pyx) with the
reference's own compiler directives (setup.py:128-131, dev/native/ExtensionHelper.py:14-20:
language_level=3, cdivision, wraparound=False, boundscheck=False, initializedcheck=False),
language=c++ and OpenMP (setup.py:104-114).  Generated C++ and the .so files go ONLY to
oracle/_ref/ (git-ignored build output).  No reference source is
copied into the repository.

Usage:  python oracle/build_ref.py            (no-op if /root/reference is absent)
"""
import os
import shutil
import sys
import sysconfig

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("URH_REFERENCE", "/root/reference")
OUT = os.path.join(HERE, "_ref")
PYX = ["signal_functions", "util", "auto_interpretation"]


def ref_available() -> bool:
    return os.path.isfile(os.path.join(REF, "src/urh/cythonext/signal_functions.pyx"))


def built() -> bool:
    suffix = sysconfig.get_config_var("EXT_SUFFIX")
    return all(os.path.isfile(os.path.join(OUT, "urh", "cythonext", m + suffix)) for m in PYX)


def build(force: bool = False) -> bool:
    if not ref_available():
        return built()
    if built() and not force:
        return True
    # The image's default CC wrapper cannot link -fopenmp (libgomp.spec missing): use /usr/bin.
    os.environ["CC"] = "/usr/bin/gcc"
    os.environ["CXX"] = "/usr/bin/g++"
    os.environ["LDSHARED"] = "/usr/bin/g++ -shared"
    import numpy as np
    from Cython.Build import cythonize
    from setuptools import Extension
    from setuptools.dist import Distribution
    from setuptools.command.build_ext import build_ext

    src_dir = os.path.join(REF, "src")
    pkg_dir = os.path.join(OUT, "urh", "cythonext")
    os.makedirs(pkg_dir, exist_ok=True)
    for d in (os.path.join(OUT, "urh"), pkg_dir):
        init = os.path.join(d, "__init__.py")
        if not os.path.exists(init):
            open(init, "w").close()
    exts = [
        Extension(
            "urh.cythonext." + m,
            [os.path.join(src_dir, "urh", "cythonext", m + ".pyx")],
            extra_compile_args=["-fopenmp", "-O2", "-Wno-cpp", "-w"],
            extra_link_args=["-fopenmp"],
            include_dirs=[np.get_include()],
            language="c++",
        )
        for m in PYX
    ]
    cwd = os.getcwd()
    os.chdir(src_dir)  # so that "urh.cythonext.util" cimports resolve; nothing is written here
    try:
        exts = cythonize(
            exts,
            build_dir=os.path.join(OUT, "_gen"),
            include_path=[src_dir],
            compiler_directives=dict(
                language_level=3, cdivision=True, wraparound=False, boundscheck=False, initializedcheck=False
            ),
            quiet=True,
        )
        dist = Distribution({"ext_modules": exts})
        cmd = build_ext(dist)
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


PYREF = os.path.join(OUT, "pyref")
# the reference's own tests that exercise the hot path without a Qt event loop (SURVEY section 4)
REF_TESTS = ["__init__.py", "utils_testing.py", "test_util.py", "test_demodulations.py", "test_modulator.py", "test_iq_array.py",
             "test_protocol_analyzer.py", "test_ringbuffer.py", "test_continuous_modulator.py", "auto_interpretation"]


def stage_python_layer(force: bool = False) -> bool:
    """Stage the reference's unmodified Python layer (src/urh/**/*.py), the hot-path test files and tests/data into
    oracle/_ref/pyref/ so that they exist on the GPU box, where /root/reference does not.  Build output like the .so
    files: git-ignored, never part of the repository.  Used by oracle/run_reference_tests.py (drop-in proof) and by
    bench.py's reference arm (the reference's own detect_center)."""
    marker = os.path.join(PYREF, ".staged")
    if not ref_available():
        return os.path.isfile(marker)
    if os.path.isfile(marker) and not force:
        return True
    shutil.rmtree(PYREF, ignore_errors=True)
    src = os.path.join(REF, "src", "urh")
    for root, dirs, files in os.walk(src):
        dirs[:] = [d for d in dirs if d not in ("__pycache__", "build")]
        rel = os.path.relpath(root, src)
        for f in files:
            if f.endswith((".py", ".txt", ".json", ".xml", ".fuzz", ".ini")) and not f.endswith((".pyx", ".pxd")):
                dst = os.path.join(PYREF, "src", "urh", rel, f)
                os.makedirs(os.path.dirname(dst), exist_ok=True)
                shutil.copy2(os.path.join(root, f), dst)
    tsrc = os.path.join(REF, "tests")
    for root, dirs, files in os.walk(tsrc):   # every test module (imports between them); only REF_TESTS are run
        dirs[:] = [d for d in dirs if d not in ("__pycache__", "data")]
        rel = os.path.relpath(root, tsrc)
        for f in files:
            if f.endswith(".py"):
                dst = os.path.join(PYREF, "tests", rel, f)
                os.makedirs(os.path.dirname(dst), exist_ok=True)
                shutil.copy2(os.path.join(root, f), dst)
    shutil.copytree(os.path.join(tsrc, "data"), os.path.join(PYREF, "tests", "data"), ignore=shutil.ignore_patterns("__pycache__"))
    open(marker, "w").write("staged from %s\n" % REF)
    return True


if __name__ == "__main__":
    ok = build(force="--force" in sys.argv)
    print("oracle/_ref built:", ok)
    print("reference python layer staged:", stage_python_layer(force="--force" in sys.argv))
    sys.exit(0 if ok or not ref_available() else 1)
