"""TEST INFRASTRUCTURE ONLY — builds the REFERENCE's own native extension (maskrcnn_benchmark/csrc: ml_nms,
modulated_deform_conv_forward, ...) for sm_90a from the reference sources (directory MQDET_REFERENCE, see
oracle/ref_loader.py) into oracle/_ref/ (git-ignored).  No reference source is copied into this repo.

    python oracle/build_ref.py

Used only by tests/test_ref_kernels_gpu.py to pin ml_nms / DCNv2 against the reference's CUDA kernels on the GPU.
"""
import glob
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("MQDET_REFERENCE", "/root/reference")
OUT = os.path.join(ROOT, "oracle", "_ref")


def main():
    csrc = os.path.join(REF, "maskrcnn_benchmark", "csrc")
    if not os.path.isdir(csrc):
        print("reference sources not present; nothing to build")
        return 0
    os.makedirs(OUT, exist_ok=True)
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0a")
    os.environ.setdefault("MAX_JOBS", "8")
    from torch.utils.cpp_extension import load
    srcs = glob.glob(os.path.join(csrc, "*.cpp")) + glob.glob(os.path.join(csrc, "cpu", "*.cpp")) + \
        glob.glob(os.path.join(csrc, "cuda", "*.cu"))
    load(name="mqdet_ref_C", sources=srcs, extra_include_paths=[csrc], build_directory=OUT, with_cuda=True,
         extra_cflags=["-DWITH_CUDA", "-O2"],
         extra_cuda_cflags=["-DWITH_CUDA", "-DCUDA_HAS_FP16=1", "-D__CUDA_NO_HALF_OPERATORS__", "-D__CUDA_NO_HALF_CONVERSIONS__",
                            "-D__CUDA_NO_HALF2_OPERATORS__", "-gencode", "arch=compute_90a,code=sm_90a"],
         is_python_module=True, verbose=False)
    print("built", glob.glob(os.path.join(OUT, "*.so")))
    return 0


if __name__ == "__main__":
    sys.exit(main())
