"""ctypes binding of the C ABI declared in include/pbb.h.

The CUDA library is the product: if ``libpbb.so`` is missing or a symbol is
absent this module raises -- there is no CPU fallback anywhere in the package.
"""
import ctypes
import os
import re
from typing import NamedTuple, Optional, Tuple

_HERE = os.path.dirname(os.path.abspath(__file__))
# PBB_LIB selects an alternative build of the same ABI (kernel-variant experiments)
LIB_PATH = os.environ.get('PBB_LIB') or os.path.join(_HERE, 'libpbb.so')

PBB_C64, PBB_C128 = 0, 1
NORM_NONE, NORM_EIGENVALUE, NORM_TRACE = 0, 1, 2
CW_NORM_1F1, CW_NORM_LOW, CW_NORM_MEDIUM, CW_NORM_HIGH, CW_NORM_TRAN_VU = range(5)
WEIGHT_TIME, WEIGHT_CONST, WEIGHT_TIED_TIME, WEIGHT_TIED, WEIGHT_FRAME = 0, 1, 2, 3, 4


class CacgmmOptions(ctypes.Structure):
    """struct pbb_cacgmm_options (include/pbb.h)."""
    _fields_ = [
        ('iterations', ctypes.c_int),
        ('covariance_norm', ctypes.c_int),
        ('weight_mode', ctypes.c_int),
        ('hermitize', ctypes.c_int),
        ('affiliation_eps', ctypes.c_double),
        ('eigenvalue_floor', ctypes.c_double),
        ('frames_per_block', ctypes.c_int),
        ('reserved', ctypes.c_int),
    ]


PBB_F32, PBB_F64 = 2, 3
PBB_I16, PBB_I32, PBB_I64 = 4, 5, 6
MASK_MAX_DIMS = 8
MASK_IDEAL_BINARY, MASK_WIENER_LIKE, MASK_IDEAL_RATIO, MASK_IDEAL_AMPLITUDE, MASK_PHASE_SENSITIVE, \
    MASK_IDEAL_COMPLEX = range(6)
ROW_SELECT_SHORT_MAX = 4096  # PBB_ROW_SELECT_SHORT_MAX


class MaskLayout(ctypes.Structure):
    """struct pbb_mask_layout (include/pbb.h)."""
    _fields_ = [
        ('nd', ctypes.c_int),
        ('reserved', ctypes.c_int),
        ('shape', ctypes.c_longlong * MASK_MAX_DIMS),
        ('in_stride', ctypes.c_longlong * MASK_MAX_DIMS),
        ('out_stride', ctypes.c_longlong * MASK_MAX_DIMS),
    ]


ND_MAX_DIMS, ND_OPERANDS = 8, 4
WEIGHT_BCAST = 8


class NdLayout(ctypes.Structure):
    """struct pbb_nd_layout (include/pbb.h)."""
    _fields_ = [
        ('nd', ctypes.c_int),
        ('reserved', ctypes.c_int),
        ('shape', ctypes.c_longlong * ND_MAX_DIMS),
        ('stride', (ctypes.c_longlong * ND_MAX_DIMS) * ND_OPERANDS),
    ]


HEADER = os.path.join(os.path.dirname(_HERE), 'include', 'pbb.h')

_SCALARS = {'int': ctypes.c_int, 'double': ctypes.c_double, 'size_t': ctypes.c_size_t,
            'long long': ctypes.c_longlong}
_STRUCTS = {'pbb_cacgmm_options': CacgmmOptions, 'pbb_mask_layout': MaskLayout, 'pbb_nd_layout': NdLayout}
# pointees passed as c_void_p; _device.call matches tensors to them by dtype
_POINTEES = ('double', 'float', 'int', 'long long', 'uint8_t', 'unsigned char', 'char', 'void')


class Param(NamedTuple):
    name: str
    ctype: object
    pointee: Optional[str]  # None for a scalar, else the C type pointed to


class Declaration(NamedTuple):
    restype: object
    params: Tuple[Param, ...]
    streamed: bool  # the last parameter is `void* stream`: a device entry point


def _c_type(spec, where):
    """'const double *' -> (ctype, pointee); ImportError for a type this binding does not know."""
    words = spec.replace('*', ' * ').split()
    stars = words.count('*')
    base = ' '.join(w for w in words if w not in ('const', '*'))
    if stars == 0 and base in _SCALARS:
        return _SCALARS[base], None
    if stars == 1 and base in _STRUCTS:
        return ctypes.POINTER(_STRUCTS[base]), base
    if stars == 1 and base in _POINTEES:
        return ctypes.c_void_p, base
    raise ImportError(f'{HEADER}: unknown C type {spec!r} in {where}')


def parse_header(path=HEADER):
    """name -> Declaration for every pbb_* function declared in include/pbb.h."""
    with open(path) as f:
        text = f.read()
    text = re.sub(r'/\*.*?\*/|//[^\n]*', ' ', text, flags=re.S)
    text = re.sub(r'^\s*#[^\n]*', ' ', text, flags=re.M)
    decls = {}
    for ret, name, args in re.findall(r'([A-Za-z_][\w\s*]*?)\s*\b(pbb_\w+)\s*\(([^()]*)\)\s*;', text):
        where = f'{" ".join(ret.split())} {name}({" ".join(args.split())})'
        ret = ' '.join(ret.replace('*', ' * ').split())
        if ret == 'void':
            restype = None
        elif ret == 'const char *':
            restype = ctypes.c_char_p
        else:
            restype, pointee = _c_type(ret, where)
            if pointee is not None:
                raise ImportError(f'{HEADER}: unknown return type in {where}')
        params = []
        if args.strip() != 'void':
            for arg in args.split(','):
                m = re.fullmatch(r'\s*(.*?)\b(\w+)\s*', arg, flags=re.S)
                if m is None or not m.group(1).strip():
                    raise ImportError(f'{HEADER}: unnamed or malformed parameter {arg.strip()!r} in {where}')
                params.append(Param(m.group(2), *_c_type(m.group(1), where)))
        streamed = bool(params) and params[-1].name == 'stream' and params[-1].pointee == 'void'
        decls[name] = Declaration(restype, tuple(params), streamed)
    return decls


DECLARATIONS = {}
_lib = None


def load():
    """Loads libpbb.so (once) and attaches the signatures parsed from include/pbb.h.  Raises ImportError with
    build instructions if the library or any declared symbol is missing, and names any declaration whose
    types it does not know."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f'{LIB_PATH} not found: the CUDA library is not built. Run '
            '`python -c "import __graft_entry__ as g; g.build()"` or '
            '`pb_bss_b200/csrc/build.sh`. There is no CPU fallback.')
    decls = parse_header()
    lib = ctypes.CDLL(LIB_PATH)
    for name, decl in decls.items():
        try:
            fn = getattr(lib, name)
        except AttributeError as e:
            raise ImportError(f'{LIB_PATH} does not export {name}; rebuild it') from e
        fn.restype = decl.restype
        fn.argtypes = [p.ctype for p in decl.params]
    DECLARATIONS.update(decls)
    _lib = lib
    return lib


class PbbError(RuntimeError):
    pass


def check(rc, what):
    """0 -> ok; < 0 -> ValueError (bad argument, LAPACK INFO<0 convention,
    cf. get_gev_vector.pyx:130-147); > 0 -> CUDA runtime failure."""
    if rc == 0:
        return
    msg = load().pbb_last_error().decode()
    if rc < 0:
        raise ValueError(f'{what}: {msg}')
    raise PbbError(f'{what}: {msg}')
