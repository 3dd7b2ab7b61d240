"""Build libd4pg_sm90.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

    python d4pg-pytorch_b200/build.py [--force] [--verbose]

The .so and the object files under csrc/_obj are build products (git-ignored).
"""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libd4pg_sm90.so")
OBJ = os.path.join(HERE, "csrc", "_obj")
SOURCES = ["abi.cu", "proj_loss.cu", "replay.cu", "obs_norm.cu", "gemm_ffma.cu", "gemm_tc.cu", "gemm_bf16.cu", "mlp_backward.cu", "mog_heads.cu", "qr_heads.cu", "adam.cu", "mlp_chain.cu", "mlp_tc_chain.cu", "learner.cu", "comm.cu", "act.cu", "param_noise.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "-Xcompiler", "-ffp-contract=off"]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def _digest(paths):
    h = hashlib.sha256()
    for p in sorted(paths):
        with open(p, "rb") as f:
            h.update(p.encode())
            h.update(f.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh"))]
    deps.append(os.path.join(os.path.dirname(HERE), "include", "d4pg_b200.h"))
    stamp = os.path.join(OBJ, "stamp")
    dig = _digest(deps)
    if not force and os.path.exists(OUT) and os.path.exists(stamp) and open(stamp).read() == dig:
        return OUT
    nvcc = _nvcc()
    procs = []
    for src in SOURCES:
        obj = os.path.join(OBJ, src.replace(".cu", ".o"))
        cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, obj, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    objs = []
    for src, obj, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode != 0:
            sys.stderr.write(out)
        if p.returncode != 0:
            raise RuntimeError("nvcc failed on %s:\n%s" % (src, out))
        objs.append(obj)
    cmd = [nvcc, "-shared", "-o", OUT] + objs + ["-lcudart", "-ldl"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n" + r.stdout)
    with open(stamp, "w") as f:
        f.write(dig)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
