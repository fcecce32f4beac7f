"""Build libdtsim.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

    python gym-duckietown_b200/build.py [--force]
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libdtsim.so")
SOURCES = ["dts_api.cu", "dts_maps.cu", "dts_kernels_logic.cu", "dts_render.cu", "dts_post.cu", "dts_state.cu", "dts_bev.cu",
           "dts_flow.cu", "dts_objects.cu", "dts_path.cu"]
# -fmad=false: no implicit FMA contraction, so fp32/fp64 arithmetic is exactly what the source says
# (the render kernels spell out fmaf() where an FMA is wanted; the CPU oracle is built the same way).
NVCC_FLAGS = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-fmad=false",
              "-Xcompiler", "-fPIC", "-shared", "-Xptxas", "-v"]


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "dtsim.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    extra = os.environ.get("DTS_NVCC_EXTRA", "").split()
    cmd = ["nvcc"] + NVCC_FLAGS + extra + ["-o", LIB] + [os.path.join(CSRC, s) for s in SOURCES] + ["-ldl"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed building libdtsim.so")
    with open(os.path.join(HERE, "build.log"), "w") as f:
        f.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
