"""In-tree build of libct2b200.so for sm_90a (cross-compiles without a GPU).

    python -m ctranslate2_b200.build [--force]

One nvcc invocation per translation unit (run in parallel), then a shared-library link against the
static CUDA runtime.  The .so lands next to this file so it travels with the repository snapshot.
"""
import concurrent.futures
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libct2b200.so")
OBJ = os.path.join(HERE, "_build")
SOURCES = [
    "kernels/rowwise.cu", "kernels/tp_rows.cu", "kernels/gemm_s8_mma.cu", "kernels/gemm_tc.cu", "kernels/gemm_decode.cu", "kernels/gemm_prefill.cu", "kernels/awq.cu", "kernels/awq_decode.cu", "kernels/awq_gemv.cu", "kernels/attention.cu", "kernels/attention_mma.cu", "kernels/attention_decode.cu",
    "kernels/decode_loop.cu", "kernels/seq2seq.cu", "kernels/whisper_align.cu", "host/engine.cc", "host/beam.cc", "host/translator.cc", "c_api.cc",
]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-O3", "-lineinfo", "-Xcompiler", "-fPIC",
         "-Xcompiler", "-fvisibility=hidden", "--expt-relaxed-constexpr", "-x", "cu"]


# No read-only-path loads (ld.global.nc): nvcc emits them for `const T* __restrict__` kernel parameters, on the promise that the
# data is not written while the kernel is alive.  Under programmatic dependent launch a kernel is alive BEFORE its producer has
# finished (it is scheduled early and blocks in griddepcontrol.wait), so the promise does not hold for activations.  The
# qualifier is therefore compiled away for device code; weights stream through TMA, so nothing that matters used that path.
NO_NC_LOADS = "-D__restrict__="
FLAGS.append(NO_NC_LOADS)

# Experimental builds beside the product library: libct2b200_<variant>.so, loaded through CT2B200_LIB.
VARIANTS = {
    "restrict": None,      # keep __restrict__ (the pre-fix behaviour), for A/B timing
}


def _deps_hash(src):
    h = hashlib.sha1()
    for root, _, files in os.walk(CSRC):
        for f in sorted(files):
            if f.endswith((".cuh", ".h")):
                h.update(open(os.path.join(root, f), "rb").read())
    h.update(open(os.path.join(HERE, "..", "include", "ct2b200.h"), "rb").read())
    h.update(open(os.path.join(CSRC, src), "rb").read())
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def _compile(src, force):
    obj = os.path.join(OBJ, src.replace("/", "_") + ".o")
    stamp = obj + ".sha1"
    digest = _deps_hash(src)
    if not force and os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == digest:
        return obj
    cmd = [NVCC] + FLAGS + ["-c", os.path.join(CSRC, src), "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
    open(stamp, "w").write(digest)
    return obj


def build(force=False, verbose=True, variant=None):
    global OUT, OBJ, FLAGS
    if variant:
        OUT = os.path.join(HERE, "libct2b200_%s.so" % variant)
        OBJ = os.path.join(HERE, "_build_" + variant)
        assert variant in VARIANTS
        FLAGS = [f for f in FLAGS if f != NO_NC_LOADS] if VARIANTS[variant] is None else FLAGS + VARIANTS[variant]
    os.makedirs(OBJ, exist_ok=True)
    with concurrent.futures.ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as ex:
        objs = list(ex.map(lambda s: _compile(s, force), SOURCES))
    newest = max(os.path.getmtime(o) for o in objs)
    if force or not os.path.exists(OUT) or os.path.getmtime(OUT) < newest:
        cmd = [NVCC, "-shared", "-o", OUT] + objs + ["-cudart", "static", "-Xlinker", "--exclude-libs,ALL"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    import ctypes
    ctypes.CDLL(OUT)          # fails here (undefined symbols) rather than on the GPU box
    if verbose:
        print("built", OUT)
    return OUT


if __name__ == "__main__":
    build(force="--force" in sys.argv,
          variant=sys.argv[sys.argv.index("--variant") + 1] if "--variant" in sys.argv else None)
