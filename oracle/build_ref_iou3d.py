"""TEST INFRASTRUCTURE ONLY -- builds the UNMODIFIED reference `iou3d_cuda` extension into oracle/_ref/.

    iou3d_cuda_ref  <- mmdet3d/ops/iou3d/src/{iou3d.cpp,iou3d_kernel.cu}

The same recipe as oracle/build_ref.py (one torch.utils.cpp_extension.load() call, CUDA cross-compiled
for sm_90a, nothing copied into this repo), kept in its own file so that the recipe of the other three
reference modules stays as it is.  GPU tests load the result with oracle.build_ref.load_ref and compare
the rotated IoU and NMS of bevfusion_b200.iou3d against the reference's own CUDA op."""
import os
import shutil
import sys

from oracle.build_ref import OUT, REF, built

NAME = "iou3d_cuda_ref"


def build(verbose=False):
    if not os.path.isdir(REF):
        return False  # GPU box: use the prebuilt file
    if built(NAME):
        return True
    os.makedirs(OUT, exist_ok=True)
    os.environ["TORCH_CUDA_ARCH_LIST"] = "9.0a"
    os.environ.setdefault("MAX_JOBS", "8")
    from torch.utils.cpp_extension import load
    src = REF + "/mmdet3d/ops/iou3d/src/"
    bdir = os.path.join("/tmp", "bevfusion_ref_build", NAME)
    os.makedirs(bdir, exist_ok=True)
    load(name=NAME, sources=[src + "iou3d.cpp", src + "iou3d_kernel.cu"], build_directory=bdir, verbose=verbose,
         with_cuda=True, is_python_module=False, extra_cflags=["-w"], extra_cuda_cflags=["-w"])
    shutil.copy(os.path.join(bdir, NAME + ".so"), os.path.join(OUT, NAME + ".so"))
    return True


if __name__ == "__main__":
    ok = build(verbose="-v" in sys.argv)
    print("built" if ok else "reference tree absent; nothing built", NAME if built(NAME) else "")
