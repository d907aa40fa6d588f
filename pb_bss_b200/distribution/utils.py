"""pb_bss/distribution/utils.py: the model containers (:118-190), their stacking and lookup helpers, and the device
kernels of ``_unit_norm`` and ``force_hermitian``."""
import difflib
import math

import numpy as np
import torch
from numpy.lib.array_utils import normalize_axis_index

from .. import _device, _lib, _nd


def get_trainer_class_from_model(parameter):
    """The trainer class of a model class or instance (utils.py:6-27), looked up in pb_bss_b200.distribution."""
    from .. import distribution
    if not hasattr(parameter, '__name__'):
        parameter = parameter.__class__
    name = parameter.__name__
    assert 'Trainer' not in name, name
    return getattr(distribution, name + 'Trainer')


def parameter_from_dict(parameter_class_or_str, d: dict):
    """A model from its ``to_dict`` (utils.py:83-115); a class name is looked up in pb_bss_b200.distribution."""
    if isinstance(parameter_class_or_str, str):
        from .. import distribution
        parameter_class_or_str = getattr(distribution, parameter_class_or_str)
    return parameter_class_or_str.from_dict(d)


class _ProbabilisticModel:
    """Dataclass mix-in: ``to_dict`` / ``from_dict`` round trip and helpful
    AttributeErrors, like the reference's base class of the same name."""

    def to_dict(self):
        out = {}
        for k in self.__dataclass_fields__.keys():
            v = getattr(self, k)
            out[k] = v.to_dict() if isinstance(v, _ProbabilisticModel) else v
        return out

    @classmethod
    def from_dict(cls, d):
        assert cls.__dataclass_fields__.keys() == d.keys(), (
            cls.__dataclass_fields__.keys(), d.keys())
        return cls(**d)

    def __getattr__(self, name):
        fields = list(self.__dataclass_fields__.keys())
        similar = difflib.get_close_matches(name, fields) or fields
        raise AttributeError(
            f'{self.__class__.__name__!r} object has no attribute {name!r}.\n'
            f'Close matches: {similar}')


_EPS_STYLES = {'plus': 0, 'max': 1, 'where': 2}


def _unit_norm(signal, *, axis=-1, eps=1e-4, eps_style='plus', ord=None):
    """signal / (vector norm along ``axis``) (utils.py:223-256), on the device (pbb_unit_norm: the norms as a
    chunked reduction, then one division pass): np.linalg.norm's vector ``ord`` (None / 2, 1, inf, -inf, 0, any other p), then eps_style
    'plus' (norm + eps), 'max' (max(norm, eps)) or 'where' (eps where the norm is 0); any other eps_style raises
    AssertionError.  Real or complex signal; integers are taken as float64 (np.linalg.norm does the same).  The norm
    is an fp64 sum in a fixed order (not NumPy's pairwise order), the quotient rounded once to the signal's dtype."""
    like = _nd.like_numpy(signal)
    x = _nd.device_view(signal)
    if isinstance(ord, str):
        raise ValueError('Invalid norm order for vectors.')
    p = 2.0 if ord is None else float(ord)
    assert eps_style in _EPS_STYLES, eps_style
    nd = x.dim()
    if nd == 0:
        raise ValueError('Improper number of dimensions to norm.')
    ax = normalize_axis_index(axis, nd)
    out = _device.empty(tuple(x.shape), x.dtype)
    rows = [a for a in range(nd) if a != ax]
    xs, os_ = x.stride(), out.stride()
    lay = _nd.layout([x.shape[a] for a in rows], [xs[a] for a in rows], [os_[a] for a in rows])
    lib = _lib.load()
    nbytes = lib.pbb_reduce_workspace_bytes(math.prod(x.shape[a] for a in rows), x.shape[ax])
    ws = _device.workspace(max(nbytes, 1))
    _device.call('pbb_unit_norm', x if x.numel() else None, _nd.CODES[x.dtype], lay, x.shape[ax], xs[ax], os_[ax], p,
                 float(eps), _EPS_STYLES[eps_style], out if out.numel() else None, ws, nbytes)
    return _device.to_host(out, like)


def stack_parameters(parameters):
    """One model whose every field is the stack of that field over ``parameters`` (utils.py:259-315); fields that
    are models are stacked the same way.  NumPy fields go through np.stack, tensor fields through torch.stack."""
    def get_type(objects):
        types = {p.__class__ for p in objects}
        assert len(types) == 1, types
        return list(types)[0]

    out_type = get_type(parameters)
    out = {}
    for k in parameters[0].__dataclass_fields__.keys():
        datas = [getattr(p, k) for p in parameters]
        get_type(datas)
        if hasattr(datas[0], '__dataclass_fields__'):
            out[k] = stack_parameters(datas)
        elif _device.is_tensor(datas[0]):
            out[k] = torch.stack(datas)
        else:
            out[k] = np.stack(datas)
    return out_type(**out)


def force_hermitian(matrix):
    """(A + A^H) / 2 over the last two axes (utils.py:318-330), one device pass (pbb_force_hermitian).  Real input
    stays real; integers are taken as float64, as NumPy's division returns."""
    like = _nd.like_numpy(matrix)
    a = _nd.device_view(matrix)
    if a.dim() < 2:
        raise np.exceptions.AxisError(-2, a.dim())
    D = a.shape[-1]
    if a.shape[-2] != D:
        raise ValueError(f'operands could not be broadcast together with shapes {tuple(a.shape)} '
                         f'{tuple(a.shape[:-2]) + (D, a.shape[-2])}')
    a = a.contiguous()
    out = _device.empty(tuple(a.shape), a.dtype)
    batch = math.prod(a.shape[:-2])
    _device.call('pbb_force_hermitian', a if a.numel() else None, _nd.CODES[a.dtype], batch, D,
                 out if out.numel() else None)
    return _device.to_host(out, like)
