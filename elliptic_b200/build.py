"""Build recipe for libelliptic_b200.so (nvcc, sm_90a only, in-tree)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "libelliptic_b200.so")
SRC = [os.path.join(HERE, "csrc", "eb200.cu"), os.path.join(HERE, "csrc", "recovery_param.cu"),
       os.path.join(HERE, "csrc", "keyset.cu"), os.path.join(HERE, "csrc", "eddsa_keyset.cu"),
       os.path.join(HERE, "csrc", "keyset_mul.cu"), os.path.join(HERE, "csrc", "eddsa_signset.cu"),
       os.path.join(HERE, "csrc", "keyset_recovery_param.cu"), os.path.join(HERE, "csrc", "x25519_keyset.cu"),
       os.path.join(HERE, "csrc", "keyset_forms.cu"), os.path.join(HERE, "csrc", "keyset_forms_nonce.cu"),
       os.path.join(HERE, "csrc", "unkeyed_forms.cu")]
DEPS = [os.path.join(HERE, "csrc", f) for f in os.listdir(os.path.join(HERE, "csrc"))] + [
    os.path.join(HERE, "..", "include", "elliptic_b200.h")]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-split-compile", "0",
              "-Xcompiler", "-fPIC", "-shared"]


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(d) > t for d in DEPS)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", LIB] + SRC
    subprocess.run(cmd, check=True)
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(LIB)
