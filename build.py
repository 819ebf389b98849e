"""Build helpers: everything is compiled IN-TREE with explicit commands, so the
package is importable from the repository tree after build().

  build_cuda()        nvcc -> go-snark-study_b200/lib/libb200snark.so   (the product: sm_90a only)
  build_gpu_arith()   nvcc -> go-snark-study_b200/lib/libb200_gpu_arith.so  (device test vehicle of the same headers)
  build_host_arith()  g++  -> go-snark-study_b200/lib/libb200_host_arith.so (CPU unit-test vehicle)
  build_oracle()      gcc  -> oracle/_build/liboracle.so             (test infrastructure)
"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.join(ROOT, "go-snark-study_b200")
CSRC = os.path.join(PKG, "csrc")
LIBDIR = os.path.join(PKG, "lib")
ORACLE = os.path.join(ROOT, "oracle")
HOSTTEST = os.path.join(ROOT, "tests", "host")     # CPU test vehicles for the kernel headers (g++, no CUDA)
DEVTEST = os.path.join(ROOT, "tests", "device")    # device test vehicles for the kernel headers (nvcc, sm_90a)

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CUDA_SOURCES = ["capi.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC", "-shared", "-Xptxas", "-v"]


def _newer(target, sources):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in sources)


def _all_sources(exts=(".cu", ".cuh", ".cpp", ".h")):
    out = []
    for d in (CSRC, os.path.join(ROOT, "include"), HOSTTEST):
        if os.path.isdir(d):
            out += [os.path.join(d, f) for f in os.listdir(d) if f.endswith(exts)]
    return out


def _run(cmd, log=None):
    p = subprocess.run(cmd, capture_output=True, text=True)
    if log:
        with open(log, "w") as f:
            f.write(" ".join(cmd) + "\n" + p.stdout + p.stderr)
    if p.returncode != 0:
        sys.stderr.write(p.stdout[-4000:] + p.stderr[-8000:])
        raise RuntimeError("build failed: " + " ".join(cmd))
    return p


def build_cuda(force=False):
    os.makedirs(LIBDIR, exist_ok=True)
    target = os.path.join(LIBDIR, "libb200snark.so")
    if not force and not _newer(target, _all_sources(exts=(".cu", ".cuh", ".h"))):   # the .cpp files are CPU test vehicles
        return target
    if not os.path.exists(NVCC):
        if os.path.exists(target):
            return target          # GPU box without a toolchain change: use the shipped build
        raise RuntimeError("nvcc not found and no prebuilt libb200snark.so")
    cmd = [NVCC, *NVCC_FLAGS, "-I", os.path.join(ROOT, "include"), "-I", CSRC,
           "-o", target, *[os.path.join(CSRC, s) for s in CUDA_SOURCES]]
    _run(cmd, log=os.path.join(LIBDIR, "nvcc_build.log"))
    return target


def build_gpu_arith(force=False):
    """nvcc build of tests/device/arith_device.cu with the product's own flags (device test vehicle for the arithmetic
    headers, tests/test_gpu_arith.py).  Not linked into libb200snark.so."""
    os.makedirs(LIBDIR, exist_ok=True)
    target = os.path.join(LIBDIR, "libb200_gpu_arith.so")
    src = os.path.join(DEVTEST, "arith_device.cu")
    if not force and not _newer(target, _all_sources(exts=(".cuh", ".h")) + [src]):
        return target
    if not os.path.exists(NVCC):
        if os.path.exists(target):
            return target          # GPU box without a toolchain change: use the shipped build
        raise RuntimeError("nvcc not found and no prebuilt libb200_gpu_arith.so")
    _run([NVCC, *NVCC_FLAGS, "-I", CSRC, "-o", target, src], log=os.path.join(LIBDIR, "nvcc_gpu_arith.log"))
    return target


def build_host_arith(force=False):
    os.makedirs(LIBDIR, exist_ok=True)
    target = os.path.join(LIBDIR, "libb200_host_arith.so")
    if not force and not _newer(target, _all_sources()):
        return target
    cmd = ["g++", "-O2", "-std=c++17", "-x", "c++", "-shared", "-fPIC", "-Wno-psabi", "-I", CSRC,
           "-o", target, os.path.join(HOSTTEST, "host_arith_test.cpp")]
    _run(cmd)
    return target


def build_host_kernels(force=False):
    """g++ build of the per-thread bucket kernels over csrc/host_stub (CPU test vehicle, tests/test_host_kernels.py)."""
    os.makedirs(LIBDIR, exist_ok=True)
    target = os.path.join(LIBDIR, "libb200_host_kernels.so")
    if not force and not _newer(target, _all_sources() + [os.path.join(HOSTTEST, "host_stub", "cuda_runtime.h")]):
        return target
    cmd = ["g++", "-O2", "-std=c++17", "-pthread", "-x", "c++", "-shared", "-fPIC", "-Wno-psabi", "-I", os.path.join(HOSTTEST, "host_stub"),
           "-I", HOSTTEST, "-I", CSRC, "-o", target, os.path.join(HOSTTEST, "host_kernel_test.cpp")]
    _run(cmd)
    return target


def build_host_fixed_base(force=False):
    """g++ build of the fixed-base kernel and its table build over csrc/host_stub (CPU test vehicle,
    tests/test_host_fixed_base.py)."""
    os.makedirs(LIBDIR, exist_ok=True)
    target = os.path.join(LIBDIR, "libb200_host_fixed_base.so")
    if not force and not _newer(target, _all_sources() + [os.path.join(HOSTTEST, "host_stub", "cuda_runtime.h")]):
        return target
    _run(["g++", "-O2", "-std=c++17", "-x", "c++", "-shared", "-fPIC", "-Wno-psabi", "-I", os.path.join(HOSTTEST, "host_stub"),
          "-I", HOSTTEST, "-I", CSRC, "-o", target, os.path.join(HOSTTEST, "fixed_base_test.cpp")])
    return target


def build_host_table_windows(force=False):
    """g++ build of the reduced-table MSM pipeline (grouped recode, grouped tails) over csrc/host_stub (CPU test vehicle,
    tests/test_host_table_windows.py)."""
    os.makedirs(LIBDIR, exist_ok=True)
    target = os.path.join(LIBDIR, "libb200_host_table_windows.so")
    if not force and not _newer(target, _all_sources() + [os.path.join(HOSTTEST, "host_stub", "cuda_runtime.h")]):
        return target
    _run(["g++", "-O2", "-std=c++17", "-pthread", "-x", "c++", "-shared", "-fPIC", "-Wno-psabi", "-I", os.path.join(HOSTTEST, "host_stub"),
          "-I", HOSTTEST, "-I", CSRC, "-o", target, os.path.join(HOSTTEST, "table_windows_test.cpp")])
    return target


def build_host_batch_msm(force=False):
    """g++ build of the batched MSM pipeline (k scalar vectors over one base set, multi-block counter scan, per-vector
    tails) over csrc/host_stub (CPU test vehicle, tests/test_host_batch_msm.py)."""
    os.makedirs(LIBDIR, exist_ok=True)
    target = os.path.join(LIBDIR, "libb200_host_batch_msm.so")
    if not force and not _newer(target, _all_sources() + [os.path.join(HOSTTEST, "host_stub", "cuda_runtime.h")]):
        return target
    _run(["g++", "-O2", "-std=c++17", "-pthread", "-x", "c++", "-shared", "-fPIC", "-Wno-psabi", "-I", os.path.join(HOSTTEST, "host_stub"),
          "-I", HOSTTEST, "-I", CSRC, "-o", target, os.path.join(HOSTTEST, "batch_msm_test.cpp")])
    return target


def build_host_prove_batch(force=False):
    """g++ build of the batched QAP front end of b200_groth16_prove_witness_batch (witness load, sparse product over k
    witnesses, batched quotients, quotient store) over csrc/host_stub (CPU test vehicle, tests/test_host_prove_batch.py)."""
    os.makedirs(LIBDIR, exist_ok=True)
    target = os.path.join(LIBDIR, "libb200_host_prove_batch.so")
    if not force and not _newer(target, _all_sources() + [os.path.join(HOSTTEST, "host_stub", "cuda_runtime.h")]):
        return target
    _run(["g++", "-O2", "-std=c++17", "-pthread", "-x", "c++", "-shared", "-fPIC", "-Wno-psabi", "-I", os.path.join(HOSTTEST, "host_stub"),
          "-I", HOSTTEST, "-I", CSRC, "-o", target, os.path.join(HOSTTEST, "prove_batch_test.cpp")])
    return target


def build_host_pinocchio_batch(force=False):
    """g++ build of the kernels of b200_pinocchio_prove_witness_batch (the quotient store into the G1T scalar vectors,
    k_pinocchio_finalize_batch) over csrc/host_stub (CPU test vehicle, tests/test_host_pinocchio_batch.py)."""
    os.makedirs(LIBDIR, exist_ok=True)
    target = os.path.join(LIBDIR, "libb200_host_pinocchio_batch.so")
    if not force and not _newer(target, _all_sources() + [os.path.join(HOSTTEST, "host_stub", "cuda_runtime.h")]):
        return target
    _run(["g++", "-O2", "-std=c++17", "-pthread", "-x", "c++", "-shared", "-fPIC", "-Wno-psabi", "-I", os.path.join(HOSTTEST, "host_stub"),
          "-I", HOSTTEST, "-I", CSRC, "-o", target, os.path.join(HOSTTEST, "pinocchio_batch_test.cpp")])
    return target


def build_host_shard_batch(force=False):
    """g++ build of the kernels of batched proving on key shards (k_groth16_finalize_batch, k_quotient_store with a
    source offset, k_pinocchio_gather_finalize_batch) over csrc/host_stub (CPU test vehicle, tests/test_host_shard_batch.py)."""
    os.makedirs(LIBDIR, exist_ok=True)
    target = os.path.join(LIBDIR, "libb200_host_shard_batch.so")
    if not force and not _newer(target, _all_sources() + [os.path.join(HOSTTEST, "host_stub", "cuda_runtime.h")]):
        return target
    _run(["g++", "-O2", "-std=c++17", "-pthread", "-x", "c++", "-shared", "-fPIC", "-Wno-psabi", "-I", os.path.join(HOSTTEST, "host_stub"),
          "-I", HOSTTEST, "-I", CSRC, "-o", target, os.path.join(HOSTTEST, "shard_batch_test.cpp")])
    return target


def build_host_short_z(force=False):
    """g++ build of the quotient by len(Z) = n (circuits with m = n + 1 signals: k_short_z_lambda, k_short_z_dot,
    k_quotient_store_shifted after the batched front end) over csrc/host_stub (CPU test vehicle, tests/test_host_short_z.py)."""
    os.makedirs(LIBDIR, exist_ok=True)
    target = os.path.join(LIBDIR, "libb200_host_short_z.so")
    if not force and not _newer(target, _all_sources() + [os.path.join(HOSTTEST, "host_stub", "cuda_runtime.h")]):
        return target
    _run(["g++", "-O2", "-std=c++17", "-pthread", "-x", "c++", "-shared", "-fPIC", "-Wno-psabi", "-I", os.path.join(HOSTTEST, "host_stub"),
          "-I", HOSTTEST, "-I", CSRC, "-o", target, os.path.join(HOSTTEST, "short_z_test.cpp")])
    return target


def build_host_setup_key(force=False):
    """g++ build of the setup into a resident key (the generator table, minting into a base set's row 0, the window rows
    from it, and the per-rank set plans) over csrc/host_stub (CPU test vehicle, tests/test_host_setup_key.py)."""
    os.makedirs(LIBDIR, exist_ok=True)
    target = os.path.join(LIBDIR, "libb200_host_setup_key.so")
    if not force and not _newer(target, _all_sources() + [os.path.join(HOSTTEST, "host_stub", "cuda_runtime.h")]):
        return target
    _run(["g++", "-O2", "-std=c++17", "-x", "c++", "-shared", "-fPIC", "-Wno-psabi", "-I", os.path.join(HOSTTEST, "host_stub"),
          "-I", HOSTTEST, "-I", CSRC, "-o", target, os.path.join(HOSTTEST, "setup_key_test.cpp")])
    return target


def build_host_verify_batch(force=False):
    """g++ build of the batched Groth16 verifier's kernels (split pairings, G2 subgroup test, classification) and of its
    aggregate stage through verify_host.cuh over csrc/host_stub (CPU test vehicle, tests/test_host_verify_batch.py)."""
    os.makedirs(LIBDIR, exist_ok=True)
    target = os.path.join(LIBDIR, "libb200_host_verify_batch.so")
    if not force and not _newer(target, _all_sources() + [os.path.join(HOSTTEST, "host_stub", "cuda_runtime.h")]):
        return target
    _run(["g++", "-O2", "-std=c++17", "-pthread", "-x", "c++", "-shared", "-fPIC", "-Wno-psabi", "-I", os.path.join(HOSTTEST, "host_stub"),
          "-I", HOSTTEST, "-I", CSRC, "-o", target, os.path.join(HOSTTEST, "verify_batch_test.cpp")])
    return target


def build_host_pinocchio_verify_batch(force=False):
    """g++ build of the batched Pinocchio verifier's classification kernel and of its aggregate stage (the reference sums
    S_i and T_i included) through verify_host.cuh over csrc/host_stub (CPU test vehicle,
    tests/test_host_pinocchio_verify_batch.py)."""
    os.makedirs(LIBDIR, exist_ok=True)
    target = os.path.join(LIBDIR, "libb200_host_pinocchio_verify_batch.so")
    if not force and not _newer(target, _all_sources() + [os.path.join(HOSTTEST, "host_stub", "cuda_runtime.h")]):
        return target
    _run(["g++", "-O2", "-std=c++17", "-pthread", "-x", "c++", "-shared", "-fPIC", "-Wno-psabi", "-I", os.path.join(HOSTTEST, "host_stub"),
          "-I", HOSTTEST, "-I", CSRC, "-o", target, os.path.join(HOSTTEST, "pinocchio_verify_batch_test.cpp")])
    return target


def build_shard_partition(force=False):
    """g++ build of csrc/shard_partition.h behind a C entry point (CPU test vehicle, tests/test_shard_partition.py)."""
    os.makedirs(LIBDIR, exist_ok=True)
    target = os.path.join(LIBDIR, "libb200_shard_partition.so")
    srcs = [os.path.join(HOSTTEST, "shard_partition_test.cpp"), os.path.join(CSRC, "shard_partition.h")]
    if not force and not _newer(target, srcs):
        return target
    _run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I", CSRC, "-o", target, srcs[0]])
    return target


def build_oracle(force=False):
    out = os.path.join(ORACLE, "_build")
    os.makedirs(out, exist_ok=True)
    target = os.path.join(out, "liboracle.so")
    srcs = [os.path.join(ORACLE, "ref_c.c")]
    if not os.path.exists(srcs[0]):
        return None
    if not force and not _newer(target, srcs):
        return target
    _run(["gcc", "-O2", "-fopenmp", "-shared", "-fPIC", "-o", target, *srcs])
    return target


if __name__ == "__main__":
    print(build_host_arith(force=True))
    print(build_oracle(force=True))
    print(build_cuda(force=True))
