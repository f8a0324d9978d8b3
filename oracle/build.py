"""Build recipes for the oracle (test infrastructure).

  build_oracle(): gcc psamask_oracle.c -> oracle/liboracle_psamask.so
  build_ref():    the reference's own lib/psa/src/cpu/{operator,psamask}.cpp compiled *where they lie* under
                  /root/reference (nothing is copied) into oracle/_ref/psamask_ref_cpu.so with
                  torch.utils.cpp_extension (the files include <torch/torch.h>, so torch's headers are needed;
                  no other external dependency, no build system of the reference is run).
  build_ref_gpu(): likewise lib/psa/src/gpu/{operator.cpp,psamask_cuda.cu} -> oracle/_ref/psamask_ref_gpu.so (nvcc
                  cross-compiles for sm_90 without a GPU): the checker of tests/test_validate_path_gpu.py and the
                  baseline of tools/bench_psamask.py.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REFERENCE = os.environ.get("SEMSEG_REFERENCE", "/root/reference")


def build_oracle():
    out = os.path.join(HERE, "liboracle_psamask.so")
    src = os.path.join(HERE, "psamask_oracle.c")
    if os.path.exists(out) and os.path.getmtime(out) >= os.path.getmtime(src):
        return out
    subprocess.check_call(["gcc", "-O2", "-fPIC", "-std=c11", "-shared", "-o", out, src])
    return out


def build_ref(verbose=False):
    """Returns the path of the built extension, or None when /root/reference is absent (GPU box)."""
    cpu_dir = os.path.join(REFERENCE, "lib", "psa", "src", "cpu")
    if not os.path.isdir(cpu_dir):
        return None
    ref_dir = os.path.join(HERE, "_ref")
    os.makedirs(ref_dir, exist_ok=True)
    for f in os.listdir(ref_dir):
        if f.startswith("psamask_ref_cpu") and f.endswith(".so"):
            return os.path.join(ref_dir, f)
    from torch.utils.cpp_extension import load
    load(name="psamask_ref_cpu",
         sources=[os.path.join(cpu_dir, "operator.cpp"), os.path.join(cpu_dir, "psamask.cpp")],
         build_directory=ref_dir, verbose=verbose)
    for f in os.listdir(ref_dir):
        if f.startswith("psamask_ref_cpu") and f.endswith(".so"):
            return os.path.join(ref_dir, f)
    raise RuntimeError("reference extension did not produce a .so in %s" % ref_dir)


def build_ref_gpu(verbose=False):
    """The reference's own CUDA extension (lib/psa/src/gpu/{operator.cpp,psamask_cuda.cu} — "the kernel the rewrite must
    beat", SURVEY.md §2.1) cross-compiled for sm_90 where the sources lie, into oracle/_ref/psamask_ref_gpu*.so. Used
    by tools/bench_psamask.py (a same-box timing of stock vs rewritten kernel) and tests/test_validate_path_gpu.py (bit
    equality). None when /root/reference is absent."""
    gpu_dir = os.path.join(REFERENCE, "lib", "psa", "src", "gpu")
    ref_dir = os.path.join(HERE, "_ref")

    def found():
        if os.path.isdir(ref_dir):
            for f in os.listdir(ref_dir):
                if f.startswith("psamask_ref_gpu") and f.endswith(".so"):
                    return os.path.join(ref_dir, f)
        return None
    if found() or not os.path.isdir(gpu_dir):
        return found()
    os.makedirs(ref_dir, exist_ok=True)
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0")
    from torch.utils.cpp_extension import load
    load(name="psamask_ref_gpu",
         sources=[os.path.join(gpu_dir, "operator.cpp"), os.path.join(gpu_dir, "psamask_cuda.cu")],
         build_directory=ref_dir, verbose=verbose, is_python_module=False)
    return found()


if __name__ == "__main__":
    print(build_oracle())
    print(build_ref(verbose="-v" in sys.argv))
    print(build_ref_gpu(verbose="-v" in sys.argv))
