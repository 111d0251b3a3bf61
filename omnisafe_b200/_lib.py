"""ctypes binding of the C-ABI library.  The prototypes are parsed from include/omnisafe_b200.h,
so the header is the single source of truth for the ABI.  There is NO CPU fallback: if the CUDA
library is missing, or a call fails, this raises."""
from __future__ import annotations

import ctypes
import os
import re

_HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(_HERE, '..', 'include', 'omnisafe_b200.h')
LIB_PATH = os.path.join(_HERE, 'lib', 'libomnisafe_b200.so')

_SCALARS = {
    'int': ctypes.c_int,
    'unsigned': ctypes.c_uint,
    'unsigned int': ctypes.c_uint,
    'float': ctypes.c_float,
    'double': ctypes.c_double,
    'long long': ctypes.c_longlong,
}


class OsbError(RuntimeError):
    pass


def parse_header(path: str = HEADER) -> dict[str, tuple[object, list[object]]]:
    """Return {name: (restype, [argtypes])} for every `osb_*` prototype in the header."""
    with open(path) as fh:
        text = fh.read()
    text = re.sub(r'/\*.*?\*/', '', text, flags=re.S)
    text = re.sub(r'//[^\n]*', '', text)
    text = re.sub(r'^\s*#[^\n]*', '', text, flags=re.M)   # preprocessor lines (include guard, constants)
    protos = {}
    for m in re.finditer(r'([A-Za-z_][\w\s\*]*?)\b(osb_\w+)\s*\(([^)]*)\)\s*;', text):
        ret, name, args = m.group(1).strip(), m.group(2), m.group(3).strip()
        restype = ctypes.c_char_p if '*' in ret else _SCALARS[ret.replace('const', '').strip()]
        argtypes = []
        if args and args != 'void':
            for a in args.split(','):
                a = a.strip()
                if '*' in a:
                    argtypes.append(ctypes.c_void_p)
                else:
                    ty = re.sub(r'\bconst\b', '', a).strip()
                    ty = ' '.join(ty.split()[:-1])  # drop the parameter name
                    argtypes.append(_SCALARS[ty])
        protos[name] = (restype, argtypes)
    return protos


class _Lib:
    def __init__(self) -> None:
        if not os.path.exists(LIB_PATH):
            raise OsbError(
                f'{LIB_PATH} not found: build it with `python -m omnisafe_b200.build` '
                '(there is no CPU fallback for the omnisafe_b200 hot path)',
            )
        self._dll = ctypes.CDLL(LIB_PATH)
        self._protos = parse_header()
        for name, (restype, argtypes) in self._protos.items():
            fn = getattr(self._dll, name)  # AttributeError if the .so does not export it
            fn.restype = restype
            fn.argtypes = argtypes
        self._checked = {
            name for name, (restype, _) in self._protos.items() if restype is ctypes.c_int
        }

    def symbols(self) -> list[str]:
        return sorted(self._protos)

    def __getattr__(self, name: str):
        fn = getattr(self._dll, name)
        # size / version queries return their value; everything else returns an error code
        if name.endswith(('_blocks', '_doubles', '_version', '_count')) or name not in self._checked:
            return fn

        def checked(*args):
            rc = fn(*args)
            if rc != 0:
                raise OsbError(f'{name} failed (rc={rc}): {self._dll.osb_last_error().decode()}')
            return rc

        checked.__name__ = name
        return checked


_LIB: _Lib | None = None


def lib() -> _Lib:
    global _LIB
    if _LIB is None:
        _LIB = _Lib()
    return _LIB


def ptr(t) -> int:
    """Device pointer of a contiguous torch tensor (0 for None)."""
    if t is None:
        return 0
    assert t.is_contiguous(), 'tensor must be contiguous'
    return t.data_ptr()


def current_stream() -> int:
    import torch  # noqa: PLC0415

    return torch.cuda.current_stream().cuda_stream
