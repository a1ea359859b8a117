"""Host builds of product headers for the CPU tests: tests/host/<name>.cpp compiled by g++ against m-loam_b200/csrc, once-rounded like
the device code (-ffp-contract=off).  Each library goes into the temporary directory under a name keyed by the hash of its source, the
product headers and the flags, so the tree is never written and an edited header gets a new library."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "m-loam_b200", "csrc")
CXXFLAGS = ["-std=c++17", "-O2", "-ffp-contract=off", "-fno-fast-math", "-shared", "-fPIC", "-I" + CSRC]
_libs = {}


def load(name: str):
    if name not in _libs:
        src = os.path.join(HERE, "host", name + ".cpp")
        h = hashlib.sha256(" ".join(CXXFLAGS).encode())
        for f in [src] + sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))):
            with open(f, "rb") as fh:
                h.update(os.path.basename(f).encode() + fh.read())
        so = os.path.join(tempfile.gettempdir(), f"mloam_{name}_{os.getuid()}_{h.hexdigest()[:16]}.so")
        if not os.path.exists(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            out = subprocess.run(["g++", *CXXFLAGS, src, "-o", tmp], capture_output=True, text=True)
            assert out.returncode == 0, out.stderr[-3000:]
            os.replace(tmp, so)
        _libs[name] = C.CDLL(so)
    return _libs[name]
