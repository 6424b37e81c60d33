"""The binding of the host builds (tests/hostbuild.py): every hc_* function a harness exports is typed from its source,
each harness is compiled once per process, and a C type the table does not know is refused."""
import ctypes as c
import glob
import os
import subprocess

import pytest

from tests import hostbuild

HARNESSES = sorted(os.path.basename(f)[:-len("_host.cpp")] for f in glob.glob(os.path.join(hostbuild.HC, "*_host.cpp"))
                   if not f.endswith("ctx_memory_host.cpp"))      # an executable against fake CUDA calls, not a library


def test_emu_names_harnesses():
    assert set(hostbuild.EMU) <= set(HARNESSES)


@pytest.mark.parametrize("name", HARNESSES)
def test_typed_functions_are_the_exported_ones(name):
    lib = hostbuild.load(name)
    nm = subprocess.run(["nm", "-D", "--defined-only", hostbuild.build(name)], capture_output=True, text=True, check=True).stdout
    exported = {line.split()[-1] for line in nm.splitlines() if line.split()[-1].startswith("hc_")}
    typed = hostbuild.functions(name)
    assert exported and set(typed) == exported
    for fn, (res, args) in typed.items():
        assert getattr(lib, fn).restype is res and getattr(lib, fn).argtypes == args, fn


@pytest.mark.parametrize("name", HARNESSES)
def test_a_harness_is_compiled_once_per_process(name, monkeypatch):
    lib, path = hostbuild.load(name), hostbuild.build(name)

    def no_compile(*a, **k):
        raise AssertionError(f"{name} compiled again")
    monkeypatch.setattr(hostbuild.subprocess, "check_call", no_compile)
    assert hostbuild.load(name) is lib and hostbuild.build(name) == path
    assert not path.startswith(hostbuild.ROOT + os.sep)


def test_prototypes_read_the_c_spellings():
    src = """
    // int hc_commented(int a) { }
    extern "C" int hc_a(const uint8_t* img, int n, unsigned seed, uint32_t s, int64_t i, long long j, uint64_t k,
                        double d, float f /* a comment */, const double* const* pp) { return 0; }
    extern "C" {
    void* hc_b() { return 0; }
    void hc_c(void) { hc_a(0, 0, 0, 0, 0, 0, 0, 0, 0, 0); }
    }"""
    assert hostbuild.prototypes(src) == {
        "hc_a": (c.c_int, [c.c_void_p, c.c_int, c.c_uint, c.c_uint, c.c_int64, c.c_int64, c.c_uint64, c.c_double, c.c_float, c.c_void_p]),
        "hc_b": (c.c_void_p, []), "hc_c": (None, [])}


@pytest.mark.parametrize("src", ['extern "C" int hc_x(size_t n) { return 0; }', 'extern "C" short hc_x(int n) { return 0; }',
                                 'extern "C" int hc_x(unsigned long n) { return 0; }'])
def test_an_unknown_c_type_raises(src):
    with pytest.raises(ValueError, match="no ctypes type"):
        hostbuild.prototypes(src)
