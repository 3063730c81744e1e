"""Build libinterdiff_b200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libinterdiff_b200.so")
SOURCES = ["api.cu", "gemm.cu", "gemm_wgmma.cu", "denoiser.cu", "sampler.cu", "lbs.cu", "geometry.cu", "correction.cu", "pointnet.cu", "metrics.cu", "rollout.cu", "skeleton_condition.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-v"]


def _stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "interdiff_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not _stale():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objs = []
    procs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    for src in SOURCES:
        obj = os.path.join(HERE, "build", src.replace(".cu", ".o"))
        objs.append(obj)
        cmd = [nvcc, "-c", os.path.join(CSRC, src), "-o", obj] + NVCC_FLAGS
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    log = []
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        log.append("== %s\n%s" % (src, out))
        failed |= p.returncode != 0
    with open(os.path.join(HERE, "build", "nvcc.log"), "w") as f:
        f.write("\n".join(log))
    if failed or verbose:
        sys.stderr.write("\n".join(log))
    if failed:
        raise RuntimeError("nvcc failed; see interdiff_b200/build/nvcc.log")
    cmd = [nvcc, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-lcudart"]
    subprocess.check_call(cmd)
    return LIB


def build_tools():
    """Stand-alone micro-benchmarks under profiles/ (not part of the library): the cluster-exchange benchmark."""
    src = os.path.join(HERE, "..", "profiles", "dsmem_bench.cu")
    out = os.path.join(HERE, "build", "dsmem_bench")
    if not os.path.exists(src) or (os.path.exists(out) and os.path.getmtime(out) >= os.path.getmtime(src)):
        return out
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-o", out, src])
    return out


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
