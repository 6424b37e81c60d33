"""The host builds of the device code, tests/hostcheck/<name>_host.cpp, as ctypes libraries: the g++ recipes, one build
per harness and recipe per process, and the typing of every hc_* function from the harness source.

Recipes:
* model: plain host code, the arithmetic headers the kernels share with the host.
* emu: the SIMT emulator (simt_emu.h) and every other harness that includes CUDA headers or needs
  -fno-strict-aliasing.  Not used for the model harnesses: -fno-strict-aliasing changes their machine code.
* tsan: the emu flags under ThreadSanitizer.  Such a library only loads in a process that has libtsan preloaded
  (tsan_env), so build() returns its path and nothing here loads it.

The libraries go to one temporary directory per process, removed at exit; nothing is written under the repository."""
import atexit
import ctypes
import functools
import os
import re
import shutil
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HC = os.path.join(ROOT, "tests", "hostcheck")
CUDA_INC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")

_EMU = ["-std=c++20", "-O2", "-ffp-contract=off", "-fno-strict-aliasing", "-pthread", "-I" + CUDA_INC, "-Wno-attributes",
        "-Wno-unknown-pragmas"]
RECIPES = {
    "model": ["-std=c++17", "-O2", "-ffp-contract=off"],
    "emu": _EMU,
    "tsan": [f for f in _EMU if f != "-O2"] + ["-O1", "-g", "-fsanitize=thread", "-Wno-tsan"],
}
EMU = ("blob_emu", "blob_large_holes", "match_emu", "fused_emu", "ba_dev_emu", "ba_batch_emu", "ba_parts", "preproc")

# the C spellings the harnesses' hc_* functions use; any pointer is c_void_p
_CTYPES = {"int": ctypes.c_int, "unsigned": ctypes.c_uint, "uint32_t": ctypes.c_uint, "int64_t": ctypes.c_int64,
           "long long": ctypes.c_int64, "uint64_t": ctypes.c_uint64, "double": ctypes.c_double, "float": ctypes.c_float}
_DEF = re.compile(r"^[ \t]*(?:extern\s+\"C\"\s+)?((?:[A-Za-z_]\w*[\s*]+)+?)(hc_\w+)\s*\(([^)]*)\)\s*\{", re.M)


def source(name):
    return os.path.join(HC, f"{name}_host.cpp")


def _ctype(spelling, ret=False):
    if "*" in spelling:
        return ctypes.c_void_p
    words = " ".join(w for w in spelling.split() if w != "const")
    if ret and words == "void":
        return None
    if words not in _CTYPES:
        raise ValueError(f"no ctypes type for the C type {spelling.strip()!r}")
    return _CTYPES[words]


def prototypes(text):
    """{hc_name: (restype, argtypes)} of the hc_* functions a harness source defines."""
    text = re.sub(r"//[^\n]*|/\*.*?\*/", " ", text, flags=re.S)
    out = {}
    for ret, name, params in _DEF.findall(text):
        args = []
        for param in params.split(","):
            param = param.strip()
            if param in ("", "void"):
                continue
            named = re.fullmatch(r"(.*?[\s*])\s*[A-Za-z_]\w*", param)
            args.append(_ctype(named.group(1) if named else param))
        out[name] = (_ctype(ret, ret=True), args)
    return out


def _text(path):
    """A source with the harness sources it #includes inlined (blob_large_holes builds on blob_emu)."""
    with open(path) as f:
        return re.sub(r'^#include "(\w+\.cpp)"', lambda m: _text(os.path.join(HC, m.group(1))), f.read(), flags=re.M)


def functions(name):
    """prototypes() of harness `name`: every hc_* function its library exports."""
    return prototypes(_text(source(name)))


def bind(lib, name):
    """Sets restype and argtypes of every hc_* function of harness `name` on the loaded library `lib`."""
    for fn, (res, args) in functions(name).items():
        getattr(lib, fn).restype, getattr(lib, fn).argtypes = res, args
    return lib


@functools.cache
def _outdir():
    d = tempfile.mkdtemp(prefix="hostbuild-")
    atexit.register(shutil.rmtree, d, True)
    return d


def build(name, tsan=False):
    """The path of harness `name` compiled under its recipe (emu for EMU, model otherwise), or under tsan."""
    return _compile(name, "tsan" if tsan else "emu" if name in EMU else "model")


@functools.cache
def _compile(name, recipe):
    out = os.path.join(_outdir(), f"lib{name}_{recipe}.so")
    subprocess.check_call(["g++", *RECIPES[recipe], "-shared", "-fPIC", "-o", out, source(name)] + (["-lm"] if recipe == "model" else []))
    return out


@functools.cache
def load(name):
    """The typed library of harness `name`, built and loaded once per process."""
    return bind(ctypes.CDLL(build(name)), name)


def ptr(a):
    """A numpy array's data pointer; None is NULL."""
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def tsan_env(tmp_path, suppressions):
    """The environment of a subprocess that runs a tsan build: libtsan preloaded, races reported without failing the
    process, `suppressions` (lines of a suppressions file) applied.  Skips the test where gcc has no libtsan."""
    import pytest
    tsan = subprocess.run(["gcc", "-print-file-name=libtsan.so"], capture_output=True, text=True).stdout.strip()
    if not tsan or not os.path.isabs(tsan) or not os.path.exists(tsan):
        pytest.skip("libtsan not available")
    supp = os.path.join(str(tmp_path), "tsan_suppressions.txt")
    with open(supp, "w") as f:
        f.write("".join(line + "\n" for line in suppressions))
    return dict(os.environ, LD_PRELOAD=tsan, TSAN_OPTIONS=f"report_signal_unsafe=0 history_size=4 exitcode=0 suppressions={supp}")
