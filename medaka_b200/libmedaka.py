"""cffi binding of libmedaka_b200.so - the counterpart of the reference's ``libmedaka`` module.

The reference builds ``libmedaka`` by cdef()-ing its C headers minus the preprocessor
lines (build.py:71-82) and Python then uses ``libmedaka.ffi`` / ``libmedaka.lib``
(medaka/features.py:64,240; medaka/common.py:29-35).  This module does the same for
include/medaka_b200.h in ABI mode (dlopen), so the .so stays a plain C-ABI library.

The product path fails loudly: ``load()`` raises if the library has not been built
(run ``python __graft_entry__.py``) and ``check()`` turns every non-zero return code
into ``MedakaB200Error`` carrying ``mdk_last_error()``.
"""
import os
import re
import threading

import cffi

_HERE = os.path.dirname(os.path.abspath(__file__))
# MDK_LIB_PATH points the binding at another build of the same library (A/B measurements)
LIB_PATH = os.environ.get("MDK_LIB_PATH") or os.path.join(_HERE, "libmedaka_b200.so")
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "medaka_b200.h")

ffi = cffi.FFI()
lib = None
_lock = threading.Lock()


class MedakaB200Error(RuntimeError):
    """A libmedaka_b200 call returned a non-zero code."""

    def __init__(self, code, message):
        super().__init__("libmedaka_b200 error {}: {}".format(code, message))
        self.code = code


def _cdef_source():
    with open(HEADER_PATH) as fh:
        text = fh.read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    lines = []
    for line in text.splitlines():
        s = line.strip()
        if s.startswith("#define MDK_") and len(s.split()) == 3:
            lines.append(s)          # integer constants cffi understands
        elif s.startswith("#") or s.startswith('extern "C"') or s == "}":
            continue
        else:
            lines.append(line)
    return "\n".join(lines)


def declared_functions():
    """Names of every function include/medaka_b200.h declares (used by the CPU symbol test)."""
    src = _cdef_source()
    return sorted(set(re.findall(r"\b(mdk_[a-z0-9_]+)\s*\(", src)))


def load():
    """dlopen the library (no GPU needed) and return ``lib``."""
    global lib
    with _lock:
        if lib is not None:
            return lib
        if not os.path.exists(LIB_PATH):
            raise MedakaB200Error(
                -100, "{} not found: build it with `python __graft_entry__.py` "
                "(there is no CPU fallback)".format(LIB_PATH))
        ffi.cdef(_cdef_source())
        lib = ffi.dlopen(LIB_PATH)
        return lib


def check(rc):
    if rc != 0:
        raise MedakaB200Error(rc, ffi.string(lib.mdk_last_error()).decode())


def device_count():
    load()
    n = ffi.new("int *")
    rc = lib.mdk_device_count(n)
    if rc != 0:
        return 0
    return int(n[0])


def require_gpu(device=0):
    """Raise unless a Hopper (sm_90) device is present - the hot path has no other backend."""
    load()
    n = device_count()
    if n <= device:
        raise MedakaB200Error(-101, "no CUDA device {} (found {}); medaka_b200 has no CPU fallback".format(device, n))
    arch = ffi.new("int *")
    sms = ffi.new("int *")
    mem = ffi.new("size_t *")
    check(lib.mdk_device_info(device, arch, sms, mem))
    if arch[0] != 90:
        raise MedakaB200Error(-102, "device {} is sm_{}; libmedaka_b200 is sm_90a only".format(device, arch[0]))
    return {"sm_arch": int(arch[0]), "sm_count": int(sms[0]), "total_mem": int(mem[0])}
