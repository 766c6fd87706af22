"""Build libp2m_b200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

    python -m pose2mesh_release_b200.build [--force]
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libp2m_b200.so")
SOURCES = ["p2m_api.cu", "kernels_simt.cu", "cheb_umma.cu", "metrics.cu", "body_model.cu", "camera.cu", "temporal.cu",
           "fscore.cu", "render.cu", "posenet.cu", "front_back.cu", "targets.cu", "inputs.cu", "optim.cu", "graph_host.cpp"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC"]
if os.environ.get("P2M_TRACE") == "1":  # debug build: per-role event timeline of the tensor-core conv kernel (tools/umma_trace.py)
    FLAGS.append("-DP2M_UMMA_TRACE")


def _stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "p2m_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not _stale():
        return LIB
    srcs = [os.path.join(CSRC, f) for f in SOURCES]
    missing = [s for s in srcs if not os.path.exists(s)]
    if missing:  # a library without them would fail only when its symbols are looked up
        raise FileNotFoundError("listed sources missing: " + ", ".join(missing))
    objs = []
    procs = []
    for src in srcs:
        obj = os.path.splitext(src)[0] + ".o"
        objs.append(obj)
        cmd = [NVCC, *FLAGS, "-c", src, "-o", obj]
        if verbose:
            cmd[1:1] = ["-Xptxas", "-v"]
        procs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for cmd, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode != 0:
            sys.stderr.write(out)
        if p.returncode != 0:
            raise RuntimeError("nvcc failed: " + " ".join(cmd))
    cmd = [NVCC, "-shared", "-o", LIB, *objs, "-gencode", "arch=compute_90a,code=sm_90a"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("link failed: " + " ".join(cmd))
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
