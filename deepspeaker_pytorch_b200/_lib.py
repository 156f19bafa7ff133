"""ctypes binding of libdsk.so, read from the C ABI in include/dsk.h, and the in-tree nvcc build recipe.

The product path has no fallback: if the shared library is missing or an entry point fails, a
RuntimeError is raised (north star: "no CPU fallback, no multi-backend dispatch").
"""
from __future__ import annotations

import ctypes
import os
import re
import shutil
import subprocess
from ctypes import POINTER, c_char_p, c_double, c_float, c_int32, c_int64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
LIB_DIR = os.path.join(_HERE, "lib")
LIB_PATH = os.path.join(LIB_DIR, "libdsk.so")
INCLUDE = os.path.join(os.path.dirname(_HERE), "include")
HEADER = os.path.join(INCLUDE, "dsk.h")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "--shared", "-Xcompiler", "-fPIC",
]


def _sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh"))) + [HEADER]


HASH_PATH = LIB_PATH + ".srchash"


def _source_hash() -> str:
    import hashlib

    h = hashlib.sha1()
    for s in _sources():
        h.update(os.path.basename(s).encode())
        with open(s, "rb") as f:
            h.update(f.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def needs_build() -> bool:
    """True when lib/libdsk.so is missing or was built from different source CONTENT (file times are not trusted:
    the tree is copied between machines, and N ranks may import it at once)."""
    if not os.path.exists(LIB_PATH):
        return True
    try:
        with open(HASH_PATH) as f:
            return f.read().strip() != _source_hash()
    except OSError:
        return True


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile csrc/*.cu for sm_90a into lib/libdsk.so (nvcc cross-compiles without a GPU).  Safe under concurrent
    callers: an exclusive file lock serialises them and the library is renamed into place."""
    if not force and not needs_build():
        return LIB_PATH
    import fcntl

    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found: cannot build libdsk.so")
    os.makedirs(LIB_DIR, exist_ok=True)
    with open(os.path.join(LIB_DIR, ".build.lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        if not force and not needs_build():  # another process built it while this one waited
            return LIB_PATH
        tmp = LIB_PATH + f".tmp{os.getpid()}"
        cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", tmp, os.path.join(CSRC, "dsk_api.cu")]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            if os.path.exists(tmp):
                os.remove(tmp)
            raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
        os.replace(tmp, LIB_PATH)
        with open(HASH_PATH, "w") as f:
            f.write(_source_hash())
        if verbose:
            print(r.stderr)
    return LIB_PATH


# ---- the binding, read from include/dsk.h at import -------------------------------------------------------------------
# The header is the only statement of the C ABI: its integer #defines and enum members become module constants
# (DSK_NUM_CONV, DSK_F16, ...), its structs ctypes Structures (dsk_weights -> DskWeights) and its prototypes the
# (restype, argtypes) pairs that load() applies.  The compiler holds csrc/dsk_api.cu to the same header.

def _ctype(decl: str, structs: dict, handles: set, where: str, ret: bool = False):
    """The ctypes type of a header type; the one place where the binding names a ctypes scalar type.  A pointer is
    c_void_p (device arrays are passed as data_ptr() integers, host out-parameters by byref() or as arrays), except a
    pointer to a header struct, to a pointer or to a handle.  ValueError naming ``where`` for any other type."""
    t = " ".join(decl.replace("*", " * ").split()).replace(" *", "*")
    if ret and t == "const char*":
        return c_char_p
    t = t.removeprefix("const ")
    if t.endswith("*"):
        pointee = t[:-1].removeprefix("const ")
        if pointee.endswith("*") or pointee in handles:
            return POINTER(c_void_p)
        return POINTER(structs[pointee]) if pointee in structs else c_void_p
    if t in handles:
        return c_void_p
    scalars = {"int32_t": c_int32, "int64_t": c_int64, "float": c_float, "double": c_double}
    if t not in scalars:
        raise ValueError(f"{where}: no ctypes type for '{t}'")
    return scalars[t]


def _declarator(decl: str, where: str):
    """(type, name, array extent or None) of a parameter or a struct field: ``const float* conv_w[DSK_NUM_CONV]``."""
    m = re.fullmatch(r"\s*(\S.*?)\s*\b(\w+)\s*(?:\[\s*(\w+)\s*\])?\s*", decl, flags=re.S)
    if not m:
        raise ValueError(f"{where}: cannot read '{' '.join(decl.split())}'")
    return m.groups()


def read_header(text: str):
    """(constants, structs, prototypes) of a C header written as include/dsk.h is.  constants: every
    ``#define DSK_<NAME> <integer>`` and enum member, by name; structs: every ``typedef struct {...} dsk_x;`` as a
    ctypes.Structure named DskX, by typedef name; prototypes: every ``ret dsk_name(params);`` as (restype, argtypes),
    by name.  ``typedef struct X* name;`` declares an opaque handle.  ValueError for anything else it meets."""
    src = re.sub(r"/\*.*?\*/|//[^\n]*", " ", text, flags=re.S)
    src = re.sub(r"#ifdef __cplusplus.*?#endif", "", src, flags=re.S)  # the extern "C" wrapper
    consts = {n: int(v) for n, v in re.findall(r"^\s*#\s*define\s+(DSK_\w+)\s+(-?\d+)\s*$", src, flags=re.M)}
    src = re.sub(r"^\s*#.*$", "", src, flags=re.M)
    for body in re.findall(r"typedef\s+enum\s*\{([^}]*)\}\s*\w+\s*;", src):
        for item in body.split(","):
            m = re.fullmatch(r"\s*(DSK_\w+)\s*=\s*(-?\d+)\s*", item)
            if not m:
                raise ValueError(f"cannot read enum member '{item.strip()}' (each needs an explicit value)")
            consts[m[1]] = int(m[2])
    handles = set(re.findall(r"typedef\s+struct\s+\w+\s*\*\s*(\w+)\s*;", src))
    structs = {}
    for body, name in re.findall(r"typedef\s+struct\s*\{([^}]*)\}\s*(\w+)\s*;", src):
        fields = []
        for field in filter(str.strip, body.split(";")):
            t, f, n = _declarator(field, name)
            t = _ctype(t, structs, handles, f"{name}.{f}")
            fields.append((f, t * (consts[n] if n in consts else int(n)) if n else t))
        camel = "".join(w.capitalize() for w in name.split("_"))
        structs[name] = type(camel, (ctypes.Structure,), {"_fields_": fields})
    *decls, rest = re.sub(r"typedef\s[^;{]*(\{[^}]*\})?[^;]*;", "", src).split(";")
    if rest.strip():
        raise ValueError(f"cannot read '{' '.join(rest.split())}'")
    prototypes = {}
    for decl in decls:
        m = re.fullmatch(r"\s*(.+?)\s*\b(dsk_\w+)\s*\((.*)\)\s*", decl, flags=re.S)
        if not m:
            raise ValueError(f"cannot read '{' '.join(decl.split())}'")
        ret, name, params = m.groups()
        params = [] if params.strip() == "void" else [_declarator(p, name)[0] for p in params.split(",")]
        prototypes[name] = (_ctype(ret, structs, handles, name, ret=True),
                            [_ctype(p, structs, handles, name) for p in params])
    return consts, structs, prototypes


with open(HEADER) as _f:
    CONSTANTS, STRUCTS, PROTOTYPES = read_header(_f.read())
globals().update(CONSTANTS)
globals().update({s.__name__: s for s in STRUCTS.values()})

_lib = None


def load() -> ctypes.CDLL:
    """Load libdsk.so (building it first if it is missing or its sources changed). Raises if unavailable — no fallback."""
    global _lib
    if _lib is not None:
        return _lib
    if needs_build():
        try:
            build()
        except Exception as e:  # a GPU box without nvcc must ship the prebuilt .so
            if not os.path.exists(LIB_PATH):
                raise RuntimeError(f"libdsk.so is missing and could not be built: {e}") from e
            if os.environ.get("DSK_STRICT_BUILD") == "1":
                raise RuntimeError(f"libdsk.so does not match csrc/ and the rebuild failed: {e}") from e
            import warnings

            warnings.warn(f"libdsk.so was built from DIFFERENT sources than csrc/ and the rebuild failed ({e}); "
                          f"loading the stale library (set DSK_STRICT_BUILD=1 to make this an error)", RuntimeWarning)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in PROTOTYPES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = load().dsk_last_error()
        raise RuntimeError(f"libdsk {what} failed ({rc}): {msg.decode() if msg else '?'}")


def cur_stream() -> int:
    import torch

    return torch.cuda.current_stream().cuda_stream


def ptr(t) -> int:
    """Raw device pointer of a tensor (None -> NULL)."""
    return 0 if t is None else t.data_ptr()
