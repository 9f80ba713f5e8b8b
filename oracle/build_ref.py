#!/usr/bin/env python
"""Build the UNMODIFIED reference native ops into oracle/_ref/ (git-ignored).

TEST / MEASUREMENT INFRASTRUCTURE ONLY.  Nothing in the product package may
import anything from oracle/.  Only tests/, __graft_entry__.smoke() and
bench.py (--impl reference / cpu_baseline) use the artefacts built here.

What is built (sources are compiled where they lie under /root/reference,
nothing is copied into the git history):

  oracle/_ref/diff_gaussian_rasterization/_C.so
        <- dgmesh/submodules/diff-gaussian-rasterization/{ext.cpp,
           rasterize_points.cu, cuda_rasterizer/{forward,backward,rasterizer_impl}.cu}
  oracle/_ref/simple_knn/_C.so
        <- dgmesh/submodules/simple-knn/{ext.cpp, spatial.cu, simple_knn.cu}

and, as the equivalent of `pip install --target` (build OUTPUT, git-ignored):

  oracle/_ref/diff_gaussian_rasterization/__init__.py   (the reference Python surface)
  oracle/_ref/refpy/{time_utils,rigid_utils,dpsr,dpsr_utils,graphics_utils}.py
        (pure-PyTorch reference modules used as MLP / DPSR / camera oracles)
  oracle/_ref/dgmesh/        the reference's whole Python tree minus submodules/ (train.py, scene/,
        utils/, arguments/, configs/): what tools/train_harness.py runs UNMODIFIED

The reference ships no sm_90a build; it needs two forced includes under gcc 13
(`<cstdint>` for rasterizer_impl.h, `<cfloat>` for simple_knn.cu) -- passed on
the command line, the sources are not patched.  We use torch's own JIT
extension builder (ninja + nvcc), not the reference's setup.py / CMake.

/root/reference does not exist on the GPU box: run this HERE; the built files
travel with the gpurun snapshot.
"""
import os
import shutil
import sys

REF = os.environ.get("DGMESH_REFERENCE", "/root/reference")
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")


def _load(name, sources, build_dir, extra_cuda, extra_inc):
    from torch.utils.cpp_extension import load
    os.makedirs(build_dir, exist_ok=True)
    load(
        name=name,
        sources=sources,
        extra_include_paths=extra_inc,
        extra_cflags=["-O3", "-include", "cstdint", "-include", "cfloat"],
        extra_cuda_cflags=["-O3", "-include", "cstdint", "-include", "cfloat",
                           "-gencode", "arch=compute_90a,code=sm_90a"] + extra_cuda,
        build_directory=build_dir,
        with_cuda=True,
        is_python_module=False,   # do not import here (no GPU needed, but keep it lazy)
        verbose=False,
    )


def build(force=False):
    if not os.path.isdir(REF):
        print(f"[build_ref] {REF} not present -- using prebuilt oracle/_ref if any")
        return os.path.isdir(OUT)
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "10.0")
    os.environ.setdefault("MAX_JOBS", "8")
    dgr = os.path.join(REF, "dgmesh/submodules/diff-gaussian-rasterization")
    knn = os.path.join(REF, "dgmesh/submodules/simple-knn")

    dgr_out = os.path.join(OUT, "diff_gaussian_rasterization")
    knn_out = os.path.join(OUT, "simple_knn")
    # each extension is built in its own process: torch's JIT builder versions the
    # module name (_C -> _C_v1) when the same name is built twice in one process
    import subprocess
    for which, out in (("dgr", dgr_out), ("knn", knn_out)):
        if force or not os.path.exists(os.path.join(out, "_C.so")):
            subprocess.check_call([sys.executable, os.path.abspath(__file__), "--one", which])
    # --- the `pip install --target` part: python surface + pure-torch modules
    shutil.copyfile(os.path.join(dgr, "diff_gaussian_rasterization/__init__.py"),
                    os.path.join(dgr_out, "__init__.py"))
    with open(os.path.join(knn_out, "__init__.py"), "w") as f:
        f.write("")
    refpy = os.path.join(OUT, "refpy")
    os.makedirs(refpy, exist_ok=True)
    for src, dst in [
        ("dgmesh/utils/time_utils.py", "time_utils.py"),
        ("dgmesh/utils/rigid_utils.py", "rigid_utils.py"),
        ("dgmesh/utils/graphics_utils.py", "graphics_utils.py"),
        ("dgmesh/utils/sh_utils.py", "sh_utils.py"),
        ("dgmesh/utils/loss_utils.py", "loss_utils.py"),
        ("dgmesh/nvdiffrast_utils/dpsr.py", "dpsr.py"),
        ("dgmesh/nvdiffrast_utils/dpsr_utils.py", "dpsr_utils.py"),
    ]:
        shutil.copyfile(os.path.join(REF, src), os.path.join(refpy, dst))
    # the reference's Python tree (train.py, scene/, utils/, arguments/, configs/ ...) for the
    # "unmodified train.py" harness (tools/train_harness.py); build output, git-ignored like the rest
    tree = os.path.join(OUT, "dgmesh")
    if os.path.isdir(tree):
        shutil.rmtree(tree)
    shutil.copytree(os.path.join(REF, "dgmesh"), tree,
                    ignore=shutil.ignore_patterns("submodules", "__pycache__", "*.so", "*.o", ".git*"))
    # remove ninja build litter (objects) to keep the snapshot small
    for d in (dgr_out, knn_out):
        for fn in os.listdir(d):
            if fn.endswith(".o") or fn.startswith(".ninja") or fn == "build.ninja":
                try:
                    os.remove(os.path.join(d, fn))
                except OSError:
                    pass
    print("[build_ref] done ->", OUT)
    return True


def _build_one(which):
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "10.0")
    os.environ.setdefault("MAX_JOBS", "8")
    dgr = os.path.join(REF, "dgmesh/submodules/diff-gaussian-rasterization")
    knn = os.path.join(REF, "dgmesh/submodules/simple-knn")
    if which == "dgr":
        _load("_C",
              [os.path.join(dgr, "ext.cpp"),
               os.path.join(dgr, "rasterize_points.cu"),
               os.path.join(dgr, "cuda_rasterizer/forward.cu"),
               os.path.join(dgr, "cuda_rasterizer/backward.cu"),
               os.path.join(dgr, "cuda_rasterizer/rasterizer_impl.cu")],
              os.path.join(OUT, "diff_gaussian_rasterization"), [], [os.path.join(dgr, "third_party/glm")])
    else:
        _load("_C",
              [os.path.join(knn, "ext.cpp"),
               os.path.join(knn, "spatial.cu"),
               os.path.join(knn, "simple_knn.cu")],
              os.path.join(OUT, "simple_knn"), [], [])


if __name__ == "__main__":
    if "--one" in sys.argv:
        _build_one(sys.argv[sys.argv.index("--one") + 1])
        sys.exit(0)
    ok = build(force="--force" in sys.argv)
    sys.exit(0 if ok else 1)
