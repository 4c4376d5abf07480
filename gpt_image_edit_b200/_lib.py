"""ctypes binding of libb2f.so (the C ABI declared in include/b2f.h).

The library is the product: there is no Python/torch fallback for any entry point.  If the
shared object is missing or a call returns a negative code, this module raises.
"""
from __future__ import annotations

import ctypes as C
import os
import re
from pathlib import Path

import torch  # noqa: F401  (loads libcudart.so.12 into the process before libb2f.so)

_HERE = Path(__file__).resolve().parent
LIB_PATH = Path(os.environ["B2F_LIB"]) if os.environ.get("B2F_LIB") else _HERE / "lib" / "libb2f.so"   # override: A/B builds
HEADER_PATH = _HERE.parent / "include" / "b2f.h"


class B2FError(RuntimeError):
    pass


def _load() -> C.CDLL:
    if not LIB_PATH.exists():
        raise B2FError(
            f"{LIB_PATH} not found: build it with `make` (or __graft_entry__.build()). "
            "There is no fallback path."
        )
    return C.CDLL(str(LIB_PATH), mode=getattr(os, "RTLD_NOW", 2))


lib = _load()


class VaeCfg(C.Structure):
    _fields_ = [("block_out", C.c_int * 4), ("layers_per_block", C.c_int), ("latent_channels", C.c_int),
                ("in_channels", C.c_int), ("out_channels", C.c_int)]


class FluxCfg(C.Structure):
    _fields_ = [(n, C.c_int) for n in (
        "num_heads", "head_dim", "num_double", "num_single", "in_channels", "out_channels",
        "joint_dim", "pooled_dim", "guidance_embeds", "mlp_ratio")]


# ctypes type of every scalar type include/b2f.h uses; pointers are c_void_p (c_char_p for char*), so ctypes
# arrays and byref() out-parameters both pass.
_SCALARS = {"int": C.c_int, "int64_t": C.c_int64, "uint64_t": C.c_uint64, "size_t": C.c_size_t,
            "float": C.c_float, "double": C.c_double, "b2f_stream_t": C.c_void_p}


def _header_text() -> str:
    return re.sub(r"/\*.*?\*/", "", HEADER_PATH.read_text(), flags=re.S)


def _ctype(decl: str, where: str):
    """ctypes type of one declared type (`const void*`, `int64_t`, `b2f_flux**`, ...); None for void."""
    words = decl.replace("*", " * ").split()
    stars = words.count("*")
    base = [w for w in words if w not in ("*", "const")]
    if len(base) != 1:
        raise B2FError(f"include/b2f.h: cannot bind type '{decl}' in {where}")
    if stars:
        return C.c_char_p if base[0] == "char" and stars == 1 else C.c_void_p
    if base[0] == "void":
        return None
    if base[0] not in _SCALARS:
        raise B2FError(f"include/b2f.h: no ctypes binding for type '{decl}' in {where}")
    return _SCALARS[base[0]]


def _signatures() -> dict:
    """{name: (restype, argtypes)} of every function prototype in include/b2f.h."""
    sigs = {}
    for ret, name, params in re.findall(r"^\s*((?:const\s+)?\w+[\s*]*?)\s*(b2f_\w+)\s*\(([^)]*)\)\s*;",
                                        _header_text(), flags=re.M):
        params = params.strip()
        args = []
        if params not in ("", "void"):
            for prm in params.split(","):
                m = re.fullmatch(r"(.*?[\s*])(\w+)", prm.strip(), flags=re.S)
                if not m:
                    raise B2FError(f"include/b2f.h: cannot parse parameter '{prm.strip()}' of {name}")
                args.append(_ctype(m.group(1), name))
        sigs[name] = (_ctype(ret, name), args)
    return sigs


_SIGNATURES = _signatures()


def declared_symbols() -> list[str]:
    """Every function name include/b2f.h declares (used by the CPU-side export test)."""
    return sorted(set(re.findall(r"\b(b2f_[a-z0-9_]+)\s*\(", _header_text())))


def _bind() -> None:
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args


_bind()


def check(code: int, what: str = "") -> None:
    if code != 0:
        msg = lib.b2f_strerror(code).decode()
        raise B2FError(f"libb2f {what} failed: {msg} (code {code})")


def stream_ptr(stream: "torch.cuda.Stream | None" = None) -> int:
    s = stream if stream is not None else torch.cuda.current_stream()
    return int(s.cuda_stream)


def ptr(t: "torch.Tensor | None") -> int | None:
    return None if t is None else int(t.data_ptr())


KERNEL_CLASSES = ("gemm", "attention", "ln_modulate", "rmsnorm_rope", "conv", "other")


def prof_enable(on: bool) -> None:
    lib.b2f_prof_enable(int(on))


def prof_collect() -> dict:
    """{class: dict(ms, launches, flops, bytes)} since the last collect (synchronises the events)."""
    out = {}
    for i, name in enumerate(KERNEL_CLASSES):
        ms, n, fl, by = C.c_double(), C.c_int64(), C.c_double(), C.c_double()
        check(lib.b2f_prof_collect(i, C.byref(ms), C.byref(n), C.byref(fl), C.byref(by)), "b2f_prof_collect")
        out[name] = dict(ms=ms.value, launches=n.value, flops=fl.value, bytes=by.value)
    return out


def prof_shapes() -> list:
    """[(tag, launches, ms, tflops)] per GEMM shape since the last call (call before prof_collect)."""
    buf = C.create_string_buffer(1 << 20)
    n = lib.b2f_prof_shapes(buf, len(buf))
    check(min(n, 0), "b2f_prof_shapes")
    out = []
    for line in buf.value.decode().splitlines():
        tag, cnt, ms, tf = line.split("\t")
        out.append((tag, int(cnt), float(ms), float(tf)))
    return out


def launch_count() -> int:
    return int(lib.b2f_launch_count())
