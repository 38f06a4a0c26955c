"""Build lepton_b200/liblepton_b200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "liblepton_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def sources():
    return sorted(os.path.join(SRC, f) for f in os.listdir(SRC) if f.endswith((".cu", ".cuh", ".cc", ".h", ".hh"))) + [
        os.path.join(os.path.dirname(HERE), "include", "lepton_b200.h")]


def needs_build():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    return any(os.path.getmtime(s) > t for s in sources())


def build(force=False, verbose=False, variant=None):
    """variant: build into lepton_b200/variants/lib<variant>.so with the LEPB200_* defines of the environment (tuning
    builds made in the build container so that no GPU time is spent compiling; selected at run time with LEPB200_LIBRARY)."""
    global OUT
    if variant:
        os.makedirs(os.path.join(HERE, "variants"), exist_ok=True)
        out = os.path.join(HERE, "variants", "lib%s.so" % variant)
        saved, OUT = OUT, out
        try:
            return _build(verbose, cli=False)
        finally:
            OUT = saved
    if not force and not needs_build():
        return OUT
    return _build(verbose, cli=True)


def _build(verbose, cli):
    cu = [os.path.join(SRC, "lep_capi.cu")]
    cc = sorted(os.path.join(SRC, f) for f in os.listdir(SRC) if f.endswith(".cc") and f != "lepton_cli.cc")
    defs = ["-D%s=%s" % (k, os.environ[k]) for k in ("LEPB200_ENC_MINBLOCKS", "LEPB200_DEC_MINBLOCKS", "LEPB200_HUFF_MINBLOCKS", "LEPB200_STREAM_HINTS") if k in os.environ]
    cmd = [NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-shared"] + defs + [
           "-Xcompiler", "-fPIC,-O3,-pthread", "-o", OUT] + cu + cc + ["-lz", "-lpthread", "-ldl"]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
        print(" ".join(cmd))
    subprocess.check_call(cmd)
    if not cli:
        return OUT
    # the `lepton`-compatible CLI over the library
    bindir = os.path.join(HERE, "bin")
    os.makedirs(bindir, exist_ok=True)
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-o", os.path.join(bindir, "lepton-b200"), os.path.join(SRC, "lepton_cli.cc"),
                           "-L" + HERE, "-llepton_b200", "-Wl,-rpath,$ORIGIN/.."])
    return OUT


if __name__ == "__main__":
    v = sys.argv[sys.argv.index("--variant") + 1] if "--variant" in sys.argv else None
    build(force="--force" in sys.argv, verbose="--quiet" not in sys.argv, variant=v)
