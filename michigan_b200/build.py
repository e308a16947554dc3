"""Build libmichigan_sm90.so (hand-written CUDA, sm_90a only) in-tree with nvcc.

    python -m michigan_b200.build [--force]

The library is a plain C-ABI shared object (include/michigan_b200.h); it does not link against torch.
nvcc cross-compiles without a GPU, so this also runs on the CPU-only build box.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB_DIR = os.path.join(HERE, "lib")
LIB_PATH = os.path.join(LIB_DIR, "libmichigan_sm90.so")
SOURCES = ["mg_api.cu", "mg_igemm.cu", "mg_aux.cu", "mg_wgrad.cu", "mg_bwd.cu", "mg_segconv.cu", "mg_peer.cu", "mg_loss.cu", "mg_conv3x3.cu", "mg_synth.cu", "mg_orient.cu", "mg_attn.cu", "mg_vgg.cu"]  # missing files are skipped
HEADERS = ["mg_ptx.cuh", "mg_internal.h", "mg_epilogue.cuh", "mg_lab.cuh", os.path.join("..", "..", "include", "michigan_b200.h")]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "--use_fast_math=false",
]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    raise RuntimeError("nvcc not found")


def _stale():
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    deps = [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    deps += [os.path.join(CSRC, h) for h in HEADERS]
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(force=False, verbose=False, probes=False):
    """Compile every CUDA source for sm_90a and link the shared library. Returns its path.
    probes=True builds the tools-only variant libmichigan_sm90_probes.so (-DMG_PROBES: what-if switches that skip work
    and the clock64() role profiles; never loaded by the product, select it with MICHIGAN_B200_LIB=<path>)."""
    lib_path = LIB_PATH.replace(".so", "_probes.so") if probes else LIB_PATH
    if not force and not probes and not _stale():
        return LIB_PATH
    os.makedirs(LIB_DIR, exist_ok=True)
    nvcc = _nvcc()
    objs = []
    procs = []
    for s in SOURCES:
        src = os.path.join(CSRC, s)
        if not os.path.exists(src):
            continue
        obj = os.path.join(LIB_DIR, s.replace(".cu", "_probes.o" if probes else ".o"))
        cmd = [nvcc, *[f for f in NVCC_FLAGS if not f.startswith("--use_fast_math")], *(["-DMG_PROBES"] if probes else []), "-c", src, "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    for cmd, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError("nvcc failed: %s\n%s" % (" ".join(cmd), out))
        if verbose and out:
            print(out)
    cmd = [nvcc, "-shared", "-o", lib_path, *objs, "-cudart", "static"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed: %s\n%s" % (" ".join(cmd), r.stdout))
    return lib_path


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv, probes="--probes" in sys.argv))
