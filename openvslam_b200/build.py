"""Builds libovs_b200.so (sm_90a, H100) in-tree with nvcc.  `python -m openvslam_b200.build`."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
SO = os.path.join(LIBDIR, "libovs_b200.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "--fmad=false",            # parity-critical float code must not be contracted (belt and braces:
                               # that code also uses __fmul_rn/__fadd_rn explicitly)
    "-Xcompiler", "-fPIC", "-Xcompiler", "-O2", "-shared",
]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cpp")))


def needs_build():
    if not os.path.exists(SO):
        return True
    t = os.path.getmtime(SO)
    # this file too: a change of NVCC_FLAGS (the target architecture) must rebuild a library built with the old flags
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "ovs_b200.h"), os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return SO
    os.makedirs(LIBDIR, exist_ok=True)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    tmp = SO + ".tmp.%d" % os.getpid()          # built next to the target, then renamed: a reader never sees a partial library
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-x", "cu"] + sources() + ["-o", tmp]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
    if res.returncode != 0:
        if os.path.exists(tmp):
            os.remove(tmp)
        raise RuntimeError("nvcc failed building libovs_b200.so")
    os.replace(tmp, SO)
    return SO


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
