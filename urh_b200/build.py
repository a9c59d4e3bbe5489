"""Build liburh_b200.so (hand-written CUDA for sm_90a + the C ABI) in-tree with nvcc.

    python -m urh_b200.build [--force]

The shared library lands next to this file (urh_b200/liburh_b200.so); it is a git-ignored build product.
"""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "liburh_b200.so")
STAMP = os.path.join(HERE, ".liburh_b200.stamp")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC,-O2,-fno-strict-aliasing,-ffp-contract=off",
    "-ccbin", "/usr/bin/g++",
    "--expt-relaxed-constexpr",
]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest():
    h = hashlib.sha256()
    for f in sorted(os.listdir(CSRC)) + []:
        with open(os.path.join(CSRC, f), "rb") as fh:
            h.update(f.encode())
            h.update(fh.read())
    with open(os.path.join(HERE, "..", "include", "urh_b200.h"), "rb") as fh:
        h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def up_to_date():
    if not os.path.isfile(LIB) or not os.path.isfile(STAMP):
        return False
    with open(STAMP) as fh:
        return fh.read().strip() == _digest()


def build_variant(name, defines):
    """experiment helper: build urh_b200/variants/liburh_b200_<name>.so with extra -D flags"""
    vdir = os.path.join(HERE, "variants")
    os.makedirs(os.path.join(vdir, "obj_" + name), exist_ok=True)
    objs = []
    for src in sources():
        obj = os.path.join(vdir, "obj_" + name, os.path.basename(src)[:-3] + ".o")
        subprocess.check_call([NVCC] + NVCC_FLAGS + ["-D" + d for d in defines] + ["-c", src, "-o", obj])
        objs.append(obj)
    out = os.path.join(vdir, "liburh_b200_%s.so" % name)
    subprocess.check_call([NVCC, "-shared", "-o", out] + objs + ["-ccbin", "/usr/bin/g++", "-lcufft", "-ldl", "-Xlinker", "-rpath,/usr/local/cuda/lib64"])
    return out


def build(force=False, verbose=False):
    if up_to_date() and not force:
        return LIB
    if not os.path.isfile(NVCC):
        if os.path.isfile(LIB):
            # prebuilt library shipped to a box without nvcc: usable only if it was built from THESE sources
            import warnings
            warnings.warn("urh_b200: nvcc not found and liburh_b200.so does not match the sources' digest (stale build?); "
                          "_lib.load_library() checks every prototype, a missing symbol fails loudly")
            return LIB
        raise RuntimeError("nvcc not found and no prebuilt liburh_b200.so")
    objs = []
    procs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    for src in sources():
        obj = os.path.join(HERE, "build", os.path.basename(src)[:-3] + ".o")
        cmd = [NVCC] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or verbose:
            sys.stderr.write("== %s\n%s\n" % (os.path.basename(src), out))
        failed = failed or p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed")
    cmd = [NVCC, "-shared", "-o", LIB] + objs + ["-ccbin", "/usr/bin/g++", "-lcufft", "-ldl", "-Xlinker", "-rpath,/usr/local/cuda/lib64"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("link failed")
    with open(STAMP, "w") as fh:
        fh.write(_digest())
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
