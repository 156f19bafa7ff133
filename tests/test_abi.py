"""The C-ABI shared library loads without a GPU and exports every symbol include/dsk.h declares, and the ctypes
binding _lib reads from that header agrees with what the C++ compiler makes of it."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest

from deepspeaker_pytorch_b200 import _lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header():
    src = open(os.path.join(ROOT, "include", "dsk.h")).read()
    return re.sub(r"/\*.*?\*/", "", src, flags=re.S)


def declared_symbols():
    return sorted(set(re.findall(r"\b(dsk_[a-z0-9_]+)\s*\(", _header())))


def declared_constants():
    src = _header()
    return sorted(set(re.findall(r"#define\s+(DSK_\w+)\s+-?\d", src)) | set(re.findall(r"\b(DSK_\w+)\s*=", src)))


def test_library_builds_and_loads():
    lib = L.load()
    assert lib.dsk_version() >= 100


def test_every_declared_symbol_is_exported_and_read_from_the_header():
    lib = L.load()
    syms = declared_symbols()
    assert len(syms) >= 15
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/dsk.h but not exported by libdsk.so"
    assert sorted(L.PROTOTYPES) == syms, "the header reader must bind exactly the declared entry points"
    assert sorted(L.CONSTANTS) == declared_constants(), "the header reader must read exactly the declared constants"


# Prints, for every entry point, the kind of its return and of each parameter (deduced from decltype, so nothing is
# linked), sizeof and offsetof of every struct field and the value of every constant.
_PROBE = r"""
#include <cstddef>
#include <cstdio>
#include <type_traits>
#include "dsk.h"

template <class T> const char* kind() {
  if constexpr (std::is_void_v<T>) return "void";
  else if constexpr (std::is_pointer_v<T>) return "ptr";
  else if constexpr (std::is_same_v<T, float>) return "f32";
  else if constexpr (std::is_same_v<T, double>) return "f64";
  else if constexpr (std::is_integral_v<T> && std::is_signed_v<T> && sizeof(T) == 4) return "i32";
  else if constexpr (std::is_integral_v<T> && std::is_signed_v<T> && sizeof(T) == 8) return "i64";
  else return "unknown";
}
template <class R, class... A> void sig(const char* name, R (*)(A...)) {
  std::printf("fn %s %s", name, kind<R>());
  (std::printf(" %s", kind<A>()), ...);
  std::printf("\n");
}
int main() {
"""


def _kind(t):
    if t is None:
        return "void"
    if t in (ctypes.c_void_p, ctypes.c_char_p) or issubclass(t, ctypes._Pointer):
        return "ptr"
    return {ctypes.c_int32: "i32", ctypes.c_int64: "i64", ctypes.c_float: "f32", ctypes.c_double: "f64"}[t]


def test_binding_matches_the_compiler(tmp_path):
    """Every restype / argtype the reader derived has the kind (pointer, 4- or 8-byte signed integer, float, double)
    that g++ gives the declaration, every Structure field the size and offset of the C field, and every constant the
    value of the C one."""
    cxx = shutil.which("g++") or shutil.which("c++") or shutil.which("clang++")
    if cxx is None:
        pytest.skip("no host C++ compiler")
    body, expected = [], []
    for name, (res, args) in sorted(L.PROTOTYPES.items()):
        body.append(f'  sig("{name}", static_cast<decltype(&{name})>(nullptr));')
        expected.append(" ".join(["fn", name, _kind(res)] + [_kind(a) for a in args]))
    for cname, S in sorted(L.STRUCTS.items()):
        body.append(f'  std::printf("struct {cname} %zu\\n", sizeof({cname}));')
        expected.append(f"struct {cname} {ctypes.sizeof(S)}")
        for field, _ in S._fields_:
            body.append(f'  std::printf("field {cname}.{field} %zu %zu\\n", sizeof({cname}::{field}), '
                        f'offsetof({cname}, {field}));')
            expected.append(f"field {cname}.{field} {getattr(S, field).size} {getattr(S, field).offset}")
    for const, value in sorted(L.CONSTANTS.items()):
        body.append(f'  std::printf("const {const} %lld\\n", static_cast<long long>({const}));')
        expected.append(f"const {const} {value}")
    src, exe = tmp_path / "probe.cc", tmp_path / "probe"
    src.write_text(_PROBE + "\n".join(body) + "\n}\n")
    r = subprocess.run([cxx, "-std=c++17", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines()
    assert got == expected


def test_header_reader_rejects_an_unknown_type():
    with pytest.raises(ValueError, match=r"dsk_bad: no ctypes type for 'size_t'"):
        L.read_header("#include <stdint.h>\nint32_t dsk_bad(size_t n);\n")


def test_sass_is_hopper_native():
    """HGMMA (wgmma) and UTMALDG/UTMASTG (TMA) must be in the shipped SASS."""
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", L.LIB_PATH], capture_output=True, text=True).stdout
    for mnem in ("HGMMA", "UTMALDG", "UTMASTG"):
        assert mnem in sass, f"{mnem} missing from libdsk.so SASS"
    assert "sm_90a" in subprocess.run([cuobjdump, "-lelf", L.LIB_PATH], capture_output=True, text=True).stdout


def test_error_convention_without_gpu():
    """No exceptions across the ABI: bad calls return a negative status and set dsk_last_error()."""
    import torch

    lib = L.load()
    h = ctypes.c_void_p()
    assert lib.dsk_create(None, 0, 0) < 0
    assert b"null" in lib.dsk_last_error()
    assert lib.dsk_create(ctypes.byref(h), 0, 7) < 0
    if not torch.cuda.is_available():
        rc = lib.dsk_create(ctypes.byref(h), 0, 0)      # no device: a CUDA error, reported not raised
        assert rc < 0 and len(lib.dsk_last_error()) > 0
        with pytest.raises(RuntimeError):
            L.check(rc, "dsk_create")
    assert lib.dsk_pairwise_distance(None, None, 0, 0, None, None) < 0
