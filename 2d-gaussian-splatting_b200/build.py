"""Builds libsurfel_b200.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

No torch headers are involved: the library is plain CUDA + a C ABI (include/surfel_rasterizer.h).
preprocess_fwd.cu is compiled with -fmad=false so that the integer-valued outputs (radii, tile
rects, sort keys) are bit-identical to the CPU oracle (see DESIGN.md, "Parity").
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB_DIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIB_DIR, "libsurfel_b200.so")
OBJ_DIR = os.path.join(HERE, "build")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "--use_fast_math=false"]
SOURCES = {
    "api.cu": [],
    "profile.cu": [],
    "preprocess_fwd.cu": ["-fmad=false"],
    "preprocess_bwd.cu": [],
    "binning.cu": [],
    "radix_sort.cu": [],
    "bucket_sort.cu": [],
    "render_fwd.cu": [],
    "render_bwd.cu": [],
    "postprocess.cu": [],
    "loss.cu": [],
    "optim.cu": [],
    "ply_pack.cu": [],
    "knn.cu": ["-fmad=false"],
    "densify.cu": ["-fmad=false"],
    "tsdf.cu": ["-fmad=false"],
    "mcubes.cu": ["-fmad=false"],
    "meshpost.cu": [],
    "chamfer.cu": ["-fmad=false"],
    "cull.cu": ["-fmad=false"],
    "metrics.cu": [],
    "camera_bwd.cu": [],
}
# Test variants of the library: one render kernel rebuilt with another batch size (slots staged per round), the rest
# shared with the main library.  tests/test_hitloop_gpu.py runs the whole hit-loop suite against each, so a change
# of the default batch sizes meets round boundaries the suite has already pinned down.
VARIANT_DIR = os.path.join(LIB_DIR, "variants")
VARIANTS = {
    "fwd_batch32": ("render_fwd.cu", ["-DSURFEL_FWD_BATCH=32"]),
    "fwd_batch64": ("render_fwd.cu", ["-DSURFEL_FWD_BATCH=64"]),
    "bwd_batch32": ("render_bwd.cu", ["-DSURFEL_BWD_BATCH=32"]),
    "bwd_batch128": ("render_bwd.cu", ["-DSURFEL_BWD_BATCH=128"]),
}


def variant_path(name):
    return os.path.join(VARIANT_DIR, f"libsurfel_{name}.so")


def _nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return "nvcc"


def _newer(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    os.makedirs(LIB_DIR, exist_ok=True)
    os.makedirs(OBJ_DIR, exist_ok=True)
    # objects and library built with other flags (another architecture, say) are rebuilt, whatever their mtimes
    stamp_path = os.path.join(OBJ_DIR, "flags.stamp")
    stamp = repr((ARCH, COMMON, SOURCES, VARIANTS))
    if not os.path.exists(stamp_path) or open(stamp_path).read() != stamp:
        force = True
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h", ".inc"))]
    headers.append(os.path.join(HERE, "..", "include", "surfel_rasterizer.h"))
    objs, procs = {}, []

    def compile_(key, src, extra, o):
        s = os.path.join(CSRC, src)
        if force or _newer(o, [s] + headers):
            cmd = [_nvcc()] + ARCH + [f for f in COMMON if f != "--use_fast_math=false"] + extra + \
                  (["-Xptxas", "-v"] if verbose else []) + ["-c", s, "-o", o]
            procs.append((key, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))

    for src, extra in SOURCES.items():
        objs[src] = os.path.join(OBJ_DIR, src.replace(".cu", ".o"))
        compile_(src, src, extra, objs[src])
    os.makedirs(os.path.join(OBJ_DIR, "variants"), exist_ok=True)
    os.makedirs(VARIANT_DIR, exist_ok=True)
    var_objs = {}
    for name, (src, flags) in VARIANTS.items():
        var_objs[name] = os.path.join(OBJ_DIR, "variants", f"{name}.o")
        compile_(name, src, SOURCES[src] + flags, var_objs[name])
    failed = False
    for key, pr in procs:
        out, _ = pr.communicate()
        if pr.returncode != 0 or verbose:
            sys.stderr.write(f"--- nvcc {key} ---\n{out}\n")
        failed |= pr.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed")
    rebuilt = {key for key, _ in procs}

    def link(target, objects):
        # link next to the target and rename: a reader (a process loading the library, a snapshot of the tree)
        # never sees a half-written file
        tmp = target + ".link"
        subprocess.check_call([_nvcc()] + ARCH + ["-shared", "-o", tmp] + objects + ["-lcudart"])
        os.replace(tmp, target)

    if force or procs or not os.path.exists(LIB):
        link(LIB, list(objs.values()))
    for name, (src, _) in VARIANTS.items():
        target = variant_path(name)
        if force or (rebuilt - {src}) or not os.path.exists(target):
            link(target, [var_objs[name] if s == src else o for s, o in objs.items()])
    with open(stamp_path, "w") as f:
        f.write(stamp)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
