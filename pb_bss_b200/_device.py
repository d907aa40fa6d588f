"""torch tensors as device-memory containers for the C ABI.

Nothing here computes: tensors are allocated, copied host<->device and handed
to the library as raw pointers on torch's current CUDA stream (``call``).
"""
import threading

import numpy as np
import torch

from . import _lib

_scope = threading.local()


class deferred_status:
    """``with deferred_status():`` -- inside the block the device status words of the library calls (non-finite
    covariances, GEV / eigensolver failures, singular systems) are not read back after every call, because each read
    synchronises the stream and exposes the launch overhead of everything that follows; they are all read when the
    block ends, in call order, and the first failing call raises what it would have raised on the spot.  Later calls of
    the block may then have run on that call's (NaN) output.  For pipelines of CUDA tensors (parallel.py)."""

    def __enter__(self):
        self.items = []
        self.prev = getattr(_scope, 'cur', None)
        _scope.cur = self
        return self

    def __exit__(self, exc_type, exc, tb):
        _scope.cur = self.prev
        if exc_type is None:
            self.check()
        return False

    def check(self):
        items, self.items = self.items, []
        for status, on_error in items:
            s = int(status.item())
            if s:
                on_error(s)


def check_status(status, on_error):
    """Read a device status word now (synchronises) or, inside ``deferred_status``, at the end of the block;
    ``on_error(s)`` raises the call's exception for a non-zero status ``s``."""
    cur = getattr(_scope, 'cur', None)
    if cur is not None:
        cur.items.append((status, on_error))
        return
    s = int(status.item())
    if s:
        on_error(s)


def require_cuda():
    if not torch.cuda.is_available():
        raise RuntimeError(
            'pb_bss_b200 needs a CUDA device (H100, sm_90a); there is no CPU '
            'fallback. torch.cuda.is_available() is False.')


def device():
    require_cuda()
    return torch.device('cuda', torch.cuda.current_device())


def is_tensor(x):
    return isinstance(x, torch.Tensor)


def to_device(x, dtype=None, keep_pinned=False):
    """numpy array / torch tensor -> contiguous CUDA tensor (copy only if needed).

    ``keep_pinned``: a contiguous CPU tensor in pinned (page-locked) memory is returned as
    it is -- the library reads such buffers in place over PCIe (include/pbb.h,
    pbb_cacgmm_fit), which overlaps the upload with the computation.
    """
    dev = device()
    if (keep_pinned and is_tensor(x) and x.device.type == 'cpu' and x.is_pinned() and x.is_contiguous()
            and (dtype is None or x.dtype == dtype)):
        return x
    if not is_tensor(x):
        x = np.asarray(x)
        if not x.flags.c_contiguous:
            x = np.ascontiguousarray(x)
        if not x.flags.writeable:
            x = x.copy()
        x = torch.from_numpy(x)
    if dtype is not None and x.dtype != dtype:
        x = x.to(dtype)
    if x.device != dev:
        x = x.to(dev, non_blocking=True)
    return x.contiguous()


def complex_dtype_code(t):
    if t.dtype == torch.complex128:
        return _lib.PBB_C128
    if t.dtype == torch.complex64:
        return _lib.PBB_C64
    raise AssertionError(f'complex input required, got {t.dtype}')


def ptr(t):
    return None if t is None else t.data_ptr()


def stream_ptr():
    return torch.cuda.current_stream().cuda_stream


_DTYPES = {'double': (torch.float64,), 'float': (torch.float32,), 'int': (torch.int32,), 'long long': (torch.int64,),
           'uint8_t': (torch.uint8, torch.bool), 'unsigned char': (torch.uint8, torch.bool), 'void': None}
_Tensor = torch.Tensor
_NUMBERS = frozenset((int, float, bool))  # isinstance(x, torch.Tensor) is slow for a non-tensor x; these skip it
_entries = {}


def _entry(name):
    """(function, arity, scalar positions, (position, dtypes) of each pointer) of a device entry point; dtypes are
    the ones a tensor may have there (None: any; an empty tuple for a struct, which takes no tensor)."""
    lib = _lib.load()
    decl = _lib.DECLARATIONS.get(name)
    if decl is None:
        raise TypeError(f'{name} is not declared in include/pbb.h')
    if not decl.streamed:
        raise TypeError(f'{name} does not take a stream; call it through _lib.load() directly')
    params = decl.params[:-1]
    scalars = tuple(i for i, p in enumerate(params) if p.pointee is None)
    pointers = tuple((i, _DTYPES.get(p.pointee, ())) for i, p in enumerate(params) if p.pointee is not None)
    _entries[name] = entry = (getattr(lib, name), len(params), scalars, pointers)
    return entry


def _placement(name, i, t, dev):
    """The current device index (looked up once per call, on the first CUDA tensor; None before) if tensor argument
    i may be passed, else raises: it must be on the current device or in pinned host memory."""
    d = t.get_device()
    if d < 0:
        if not t.is_pinned():
            raise ValueError(f'{name}: argument {i + 1} is in pageable host memory; the device cannot read it')
        return dev
    if dev is None:
        dev = torch.cuda.current_device()
    if d != dev:
        raise ValueError(f'{name}: argument {i + 1} is on cuda:{d}, the current device is cuda:{dev}')
    return dev


def call(name, *args):
    """Calls the device entry point ``name`` of include/pbb.h on the current stream and raises through _lib.check.

    ``args`` are its parameters without the stream.  A pointer takes None (NULL), a ctypes object, or a tensor
    whose dtype matches the pointee (float64 for double, float32 for float, int32 for int, int64 for long long,
    uint8 or bool for uint8_t, any for void) and that is on the current CUDA device or in pinned host memory.  A
    Python int for a pointer, or a tensor for a scalar, is a TypeError.  Contiguity is the caller's business: some
    entry points take strides.  Everything is checked before the stream is read or the library is called."""
    fn, arity, scalars, pointers = _entries.get(name) or _entry(name)
    if len(args) != arity:
        raise TypeError(f'{name} takes {arity} arguments besides the stream, got {len(args)}')
    for i in scalars:
        a = args[i]
        if type(a) not in _NUMBERS and isinstance(a, _Tensor):
            raise TypeError(f'{name}: argument {i + 1} is a scalar, got a tensor')
    cargs = list(args)
    dev = None
    for i, want in pointers:
        a = args[i]
        if a is None:
            continue
        if isinstance(a, _Tensor):
            if want is not None and a.dtype not in want:
                raise TypeError(f'{name}: argument {i + 1} wants {" or ".join(map(str, want)) or "no tensor"}, '
                                f'got {a.dtype}')
            if a.get_device() != dev:
                dev = _placement(name, i, a, dev)
            cargs[i] = a.data_ptr()
        elif isinstance(a, int):
            raise TypeError(f'{name}: argument {i + 1} is a pointer; pass a tensor, None or a ctypes object')
    _lib.check(fn(*cargs, torch.cuda.current_stream().cuda_stream), name)


def empty(shape, dtype):
    return torch.empty(shape, dtype=dtype, device=device())


def to_host(t, like_numpy):
    """Returns numpy if the caller passed numpy, else the tensor itself."""
    if like_numpy:
        return t.cpu().numpy()
    return t


_workspaces = {}


def workspace(nbytes):
    """A cached uint8 scratch tensor of at least nbytes on the current device
    (the caller of the C ABI owns all memory, include/pbb.h)."""
    dev = device()
    key = (dev.index, torch.cuda.current_stream().cuda_stream)
    ws = _workspaces.get(key)
    if ws is None or ws.numel() < nbytes:
        ws = torch.empty(int(nbytes), dtype=torch.uint8, device=dev)
        _workspaces[key] = ws
    return ws
