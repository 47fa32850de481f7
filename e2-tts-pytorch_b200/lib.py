"""ctypes binding of libb200e2tts.so, generated from include/b200_e2tts.h at import time.

The header is the single source of truth for the C ABI: every `typedef struct {...} name;` becomes a
ctypes.Structure and every `int b200_*(...)` prototype gets argtypes/restype, so the Python side cannot
drift from the library. There is NO fallback: if the shared library is missing or a call fails a
RuntimeError is raised (north star: no CPU fallback).
"""
from __future__ import annotations

import ctypes
import os
import re

_HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(os.path.dirname(_HERE), 'include', 'b200_e2tts.h')
LIB_PATH = os.environ.get('B200_LIB') or os.path.join(_HERE, 'libb200e2tts.so')   # B200_LIB: developer A/B builds of the same ABI

_SCALARS = {
    'int32_t': ctypes.c_int32, 'int64_t': ctypes.c_int64, 'uint64_t': ctypes.c_uint64, 'uint32_t': ctypes.c_uint32,
    'float': ctypes.c_float, 'int': ctypes.c_int, 'size_t': ctypes.c_size_t, 'b200_stream_t': ctypes.c_void_p,
}


def _strip_comments(src):
    src = re.sub(r'/\*.*?\*/', ' ', src, flags=re.S)
    return re.sub(r'//[^\n]*', ' ', src)


def parse_header(path=HEADER):
    """-> (structs: {name: [(field, ctype)]}, functions: {name: (restype, [ctype])})"""
    src = _strip_comments(open(path).read())
    structs = {}
    for m in re.finditer(r'typedef\s+struct\s*\{(.*?)\}\s*(\w+)\s*;', src, flags=re.S):
        fields = []
        for decl in m.group(1).split(';'):
            decl = decl.strip()
            if not decl:
                continue
            first, *rest = [p.strip() for p in decl.split(',')]
            toks = first.replace('*', ' * ').split()
            name = toks[-1]
            base = [t for t in toks[:-1] if t not in ('const', '*')]
            ptr = '*' in toks[:-1]
            fields.append((name, ctypes.c_void_p if ptr else _SCALARS[base[-1]]))
            for r in rest:
                isptr = r.startswith('*')
                fields.append((r.lstrip('* ').strip(), ctypes.c_void_p if isptr else _SCALARS[base[-1]]))
        structs[m.group(2)] = fields
    funcs = {}
    body = re.sub(r'typedef\s+struct\s*\{.*?\}\s*\w+\s*;', ' ', src, flags=re.S)
    for m in re.finditer(r'([\w\s\*]+?)\b(b200_\w+)\s*\(([^)]*)\)\s*;', body):
        ret, name, args = m.group(1).strip(), m.group(2), m.group(3).strip()
        if ret.startswith('typedef') or name == 'b200_stream_t':
            continue
        argt = []
        if args and args != 'void':
            for a in args.split(','):
                a = a.strip()
                if '*' in a:
                    argt.append(ctypes.c_void_p)
                else:
                    toks = [t for t in a.split() if t != 'const']
                    argt.append(_SCALARS[toks[0]])
        if '*' in ret:
            restype = ctypes.c_char_p
        else:
            restype = _SCALARS.get([t for t in ret.split() if t != 'const'][-1], ctypes.c_int)
        funcs[name] = (restype, argt)
    return structs, funcs


STRUCT_FIELDS, FUNCTIONS = parse_header()
STRUCTS = {name: type(name, (ctypes.Structure,), {'_fields_': fields}) for name, fields in STRUCT_FIELDS.items()}

_lib = None


def load():
    """Load the CUDA library (loudly)."""
    global _lib
    if _lib is None:
        if not os.path.isfile(LIB_PATH):
            raise RuntimeError(f'{LIB_PATH} is missing: build it with `python -c "import __graft_entry__ as g; g.build()"` '
                               f'(there is no CPU fallback for the CUDA hot path)')
        lib = ctypes.CDLL(LIB_PATH)
        for name, (restype, argt) in FUNCTIONS.items():
            fn = getattr(lib, name)  # AttributeError if the library does not export a declared symbol
            fn.restype, fn.argtypes = restype, argt
        _lib = lib
    return _lib


def last_error():
    return load().b200_last_error().decode()


_PLAIN = (int, float, bool, type(None))


def _ptr(v):
    if v.__class__ in _PLAIN:      # scalars and NULL pass through (checked first: this runs ~13k times per training step)
        return v
    if hasattr(v, 'data_ptr'):
        return v.data_ptr()
    return v


def make_args(struct_name, **kw):
    s = STRUCTS[struct_name]()
    for k, v in kw.items():
        setattr(s, k, v if v.__class__ in _PLAIN else _ptr(v))
    return s


def make_args_positional(struct_name, field_names, values):
    """Fast path for hot call sites: `values` in header field order (checked once per call site against `field_names`)."""
    cls = STRUCTS[struct_name]
    if not getattr(cls, '_order_checked_' + str(len(field_names)), False):
        declared = [f for f, _ in STRUCT_FIELDS[struct_name]][:len(field_names)]
        if declared != list(field_names):
            raise RuntimeError(f'{struct_name}: header field order {declared} != binding order {list(field_names)}')
        setattr(cls, '_order_checked_' + str(len(field_names)), True)
    return cls(*[v if v.__class__ in _PLAIN else _ptr(v) for v in values])


def call(fn_name, *args):
    """Call a C-ABI entry point; tensors are passed as raw device pointers; raises on a non-zero code."""
    lib = load()
    conv = [a if a.__class__ in _PLAIN else (ctypes.byref(a) if isinstance(a, ctypes.Structure) else _ptr(a)) for a in args]
    rc = getattr(lib, fn_name)(*conv)
    if rc != 0:
        raise RuntimeError(f'{fn_name} failed (rc={rc}): {last_error()}')


def launch_count():
    return int(load().b200_launch_count())
