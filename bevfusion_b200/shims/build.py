"""Build the four drop-in pybind modules (`bev_pool_ext`, `voxel_layer`, `sparse_conv_ext`, `iou3d_cuda`: the
names the reference's python wrappers import, mmdet3d/ops/{bev_pool,voxel,spconv,iou3d}) in-tree, linked against
libbevfusion_b200.so.  Plain C++ (no .cu): every call forwards to the C ABI."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
LIB_DIR = os.path.join(os.path.dirname(HERE), "lib")
OUT_DIR = os.path.join(LIB_DIR, "shims")
MODULES = ("bev_pool_ext", "voxel_layer", "sparse_conv_ext", "iou3d_cuda")


def so_path(name):
    return os.path.join(OUT_DIR, name + ".so")


def built(name):
    src = os.path.join(HERE, name + ".cpp")
    so = so_path(name)
    return os.path.exists(so) and os.path.getmtime(so) >= os.path.getmtime(src)


def build(force=False, verbose=False):
    from torch.utils.cpp_extension import load
    os.makedirs(OUT_DIR, exist_ok=True)
    for name in MODULES:
        if built(name) and not force:
            continue
        load(name=name, sources=[os.path.join(HERE, name + ".cpp")], build_directory=OUT_DIR,
             extra_include_paths=[os.path.join(ROOT, "include")],
             extra_cflags=["-O2", "-std=c++17"],
             extra_ldflags=["-L" + LIB_DIR, "-lbevfusion_b200", "-Wl,-rpath,'$$ORIGIN/..'", "-L/usr/local/cuda/lib64", "-lcudart"],
             with_cuda=True, is_python_module=True, verbose=verbose)
    return [so_path(n) for n in MODULES]


def load_module(name):
    """import the built extension by file path (fails loudly when it has not been built)"""
    import importlib.util
    import torch  # noqa: F401  (libtorch must be loaded first)
    path = so_path(name)
    if not os.path.exists(path):
        raise RuntimeError("%s is not built: run `python -m bevfusion_b200.shims.build`" % path)
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
