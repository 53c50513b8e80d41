"""The audio stages' test shims (tests/csrc/{resample,stretch,limit}_shim.cu): their C signatures, one build helper, and
the sizes the tests need, read from the C header and the kernels rather than restated."""
import ctypes as C
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

vp, i32, i64 = C.c_void_p, C.c_int, C.c_longlong
pi, pl, pf = C.POINTER(C.c_int), C.POINTER(C.c_longlong), C.POINTER(C.c_float)
SIGNATURES = {
    "resample_shim": {"resample_shim_poly": [i32, C.POINTER(vp), pi, pi, pi, i32, pl, pl, pi, vp, i64, vp, vp, i64],
                      "resample_shim_move": [i32, pi, pl, pi, vp, i32, vp, i32]},
    "stretch_shim": {"stretch_shim_wsola": [i32, pl, pl, pi, vp, vp, i64, vp, vp, vp, vp, i64],
                     "stretch_shim_move": [i32, pl, pl, pi, vp, vp, vp, vp, i32]},
    "limit_shim": {"limit_shim_step": [i32, pl, pl, pi, pf, vp, i64, vp, vp, i64],
                   "limit_shim_move": [i32, pi, pl, pi, pf, vp, i32, vp, i32]},
}


def _read(path, pattern):
    src = open(os.path.join(ROOT, path)).read()
    return {k: int(v) for k, v in re.findall(pattern, src)}


_HEADER = _read("include/qwen3tts_b200.h", r"#define (Q3_(?:RESAMPLE|STRETCH|LIMIT)_\w+) (\d+)\b")
_STRETCH = _read("qwen3-tts_b200/csrc/stretch_kernels.cuh", r"constexpr int (kSt\w+) = (\d+);")
RESAMPLE_HIST, RESAMPLE_ROW_BYTES = _HEADER["Q3_RESAMPLE_HIST"], _HEADER["Q3_RESAMPLE_ROW_BYTES"]
STRETCH_HIST, STRETCH_ROW_BYTES = _HEADER["Q3_STRETCH_HIST"], _HEADER["Q3_STRETCH_ROW_BYTES"]
LIMIT_HIST, LIMIT_ROW_BYTES = _HEADER["Q3_LIMIT_HIST"], _HEADER["Q3_LIMIT_ROW_BYTES"]
STRETCH_PAD, STRETCH_MAX_IN = _STRETCH["kStPad"], _STRETCH["kStMaxIn"]


def build(out_dir, names):
    """{name: CDLL} of the named shims, compiled side by side under the library's flags, with their signatures set."""
    from qwen3_tts_b200 import build as b
    procs = {n: subprocess.Popen([b._nvcc()] + b.NVCC_FLAGS + ["-shared", "-I", b.CSRC,
                                  os.path.join(ROOT, "tests", "csrc", f"{n}.cu"), "-o", os.path.join(out_dir, f"lib{n}.so")],
                                 stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True) for n in names}
    libs = {}
    for n, p in procs.items():
        log = p.communicate()[0]
        assert p.returncode == 0, f"{n} build failed:\n{log}"
        libs[n] = C.CDLL(os.path.join(out_dir, f"lib{n}.so"))
        for fn, args in SIGNATURES[n].items():
            getattr(libs[n], fn).argtypes = args
    return libs


def load(factory, name):
    """One shim, built in a fresh pytest temporary directory (a module fixture's `tmp_path_factory`)."""
    return build(str(factory.mktemp(name)), [name])[name]
