"""CPU-side checks of the drop-in boundary: the C-ABI library loads without a
GPU and exports every symbol include/pbb.h declares; host-side argument logic."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    text = open(os.path.join(ROOT, 'include', 'pbb.h')).read()
    text = re.sub(r'/\*.*?\*/', '', text, flags=re.S)
    return sorted(set(re.findall(r'\b(pbb_[a-z0-9_]+)\s*\(', text)))


def test_every_declared_symbol_is_exported_and_parsed():
    """Every pbb_* declaration of include/pbb.h is exported by the library and bound with the argtypes and restype
    parsed from the header."""
    from pb_bss_b200 import _lib
    lib = _lib.load()
    names = _declared_symbols()
    assert len(names) >= 6, names
    for n in names:
        assert hasattr(lib, n), f'{n} declared in include/pbb.h but not exported'
        assert n in _lib.DECLARATIONS, f'{n} is not parsed from include/pbb.h'
        decl = _lib.DECLARATIONS[n]
        assert getattr(lib, n).argtypes == [p.ctype for p in decl.params], n
        assert getattr(lib, n).restype is decl.restype, n
    assert set(_lib.DECLARATIONS) == set(names)


def test_version_error_string_and_workspace_size():
    from pb_bss_b200 import _lib
    lib = _lib.load()
    assert lib.pbb_version() >= 100
    assert isinstance(lib.pbb_last_error(), bytes)
    n = lib.pbb_cacgmm_workspace_bytes(513, 500, 8, 3)
    assert 513 * 500 * 8 * 16 < n < 1 << 30
    assert lib.pbb_cacgmm_workspace_bytes(0, 1, 1, 1) == 0


def test_bad_arguments_are_rejected_before_any_launch():
    """Negative return = index of the offending argument (LAPACK INFO<0 style);
    no GPU is touched for these."""
    from pb_bss_b200 import _lib
    lib = _lib.load()
    opts = _lib.CacgmmOptions(iterations=1, covariance_norm=1, weight_mode=0, hermitize=1,
                              affiliation_eps=1e-10, eigenvalue_floor=1e-10, frames_per_block=0, reserved=0)
    rc = lib.pbb_cacgmm_fit(None, 1, 1, 1, 4, 2, None, None, None, ctypes.byref(opts),
                            None, None, None, None, 0, None, None)
    assert rc == -1 and b'y is null' in lib.pbb_last_error()
    rc = lib.pbb_cacgmm_fit(1, 7, 1, 1, 4, 2, None, None, None, ctypes.byref(opts),
                            None, None, None, None, 0, None, None)
    assert rc == -2
    rc = lib.pbb_cacgmm_fit(1, 1, 1, 1, 40, 2, None, None, None, ctypes.byref(opts),
                            None, None, None, None, 0, None, None)
    assert rc == -5 and b'D < 35' in lib.pbb_last_error()
    with pytest.raises(ValueError):
        _lib.check(rc, 'pbb_cacgmm_fit')


def test_unknown_reserved_bits_are_rejected():
    """pbb_cacgmm_options.reserved: bit 0 selects the multi-kernel path, any other bit is an error of the options
    (argument 10), found before any device work; 0 and 1 pass on to the next check, the null model outputs
    (argument 11)."""
    from pb_bss_b200 import _lib
    lib = _lib.load()
    for reserved, want in ((0, -11), (1, -11), (2, -10), (3, -10), (1 << 30, -10), (-1, -10)):
        opts = _lib.CacgmmOptions(iterations=1, covariance_norm=1, weight_mode=0, hermitize=1, affiliation_eps=1e-10,
                                  eigenvalue_floor=1e-10, frames_per_block=0, reserved=reserved)
        rc = lib.pbb_cacgmm_fit(1, 1, 1, 1, 4, 2, None, None, None, ctypes.byref(opts),
                                None, None, None, None, 0, None, None)
        assert rc == want, (reserved, rc, lib.pbb_last_error())
        if want == -10:
            assert b'reserved' in lib.pbb_last_error()


def test_no_cpu_fallback_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip('GPU present')
    from pb_bss_b200.distribution import CACGMMTrainer
    y = np.ones((2, 10, 4), dtype=np.complex128)
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        CACGMMTrainer().fit(y, num_classes=2, iterations=1)


@pytest.mark.parametrize('F,I,arrive,cap', [(513, 100, 15, 467), (129, 20, 30, 292), (7, 5, 1, 292), (40, 12, 3, 10),
                                            (513, 1, 8, 292), (1, 9, 4, 4), (2000, 3, 64, 50)])
def test_streamed_task_order_is_a_valid_schedule(F, I, arrive, cap):
    """Host logic of the streamed upload (api_cacgmm.cu, build_streamed_order): every (bin, iteration) exactly
    once, (bin, it) after (bin, it - 1), bins entering in ascending (= arrival) order -- the properties the
    persistent kernel's no-deadlock argument rests on."""
    from pb_bss_b200 import _lib
    lib = _lib.load()
    order = np.zeros(F * I, dtype=np.int32)
    rc = lib.pbb_streamed_task_order(F, I, arrive, cap, order.ctypes.data_as(ctypes.POINTER(ctypes.c_int)))
    assert rc == 0
    bins, its = order & 0xffff, order >> 16
    assert bins.min() >= 0 and bins.max() == F - 1 and its.min() == 0 and its.max() == I - 1
    assert len(set(zip(bins.tolist(), its.tolist()))) == F * I
    pos = np.empty((F, I), dtype=np.int64)
    pos[bins, its] = np.arange(F * I)
    assert (np.diff(pos, axis=1) > 0).all()
    if cap >= arrive:  # then bins enter in the order in which they arrive
        assert (np.diff(pos[:, 0]) > 0).all()
    assert lib.pbb_streamed_task_order(F, 0, arrive, cap, order.ctypes.data_as(ctypes.POINTER(ctypes.c_int))) == -2


def _dispatch(F, T, D, K, lean=1, streamed=0, sms=132):
    from pb_bss_b200 import _lib
    lib = _lib.load()
    kernel, split = ctypes.c_int(-1), ctypes.c_int(-1)
    rc = lib.pbb_em_dispatch(F, T, D, K, lean, streamed, sms, ctypes.byref(kernel), ctypes.byref(split))
    assert rc == 0, lib.pbb_last_error()
    return kernel.value, split.value


def test_em_kernel_dispatch_for_the_benchmark_configs():
    """Host logic of pbb_cacgmm_fit's kernel choice (api_cacgmm.cu: choose_sticky / choose_frame_split) on a 132-SM
    GPU: 0 = task kernel em_ws, 1 = sticky bins (one cluster per bin), 2 = single-role persistent kernel."""
    assert _dispatch(513, 500, 8, 3) == (0, 1)                 # C2: more bins than CTA slots
    assert _dispatch(257, 500, 8, 3) == (0, 1)                 # C3, 2 ranks: 4 ring stages per bin do not fit one CTA
    assert _dispatch(129, 500, 8, 3) == (1, 2)                 # C3, 4 ranks
    assert _dispatch(65, 500, 8, 3) == (1, 4)                  # C3, 8 ranks
    assert _dispatch(65, 500, 8, 3, streamed=1) == (0, 4)      # pinned host input: task kernel with the frame split
    assert _dispatch(129, 200, 4, 2) == (2, 1)                 # C1: the sweep is too short to split
    assert _dispatch(257, 1000, 6, 4) == (2, 1)                # C4
    assert _dispatch(65, 1000, 6, 4) == (2, 4)
    assert _dispatch(40, 500, 8, 3, lean=0) == (2, 4)          # saliency / masks: full variant
    assert _dispatch(64, 1100, 8, 3) == (1, 4)                 # 9 ring stages: 3 per CTA
    assert _dispatch(10, 2000, 8, 3) == (0, 4)                 # 16 stages: a part does not fit the ring of a sticky CTA
    assert _dispatch(5, 100, 8, 2) == (1, 1)                   # one ring stage: nothing to split


def test_em_kernel_dispatch_invariants():
    from pb_bss_b200 import _lib
    lib = _lib.load()
    rng = np.random.default_rng(0)
    for _ in range(300):
        F, T = int(rng.integers(1, 2000)), int(rng.integers(2, 3000))
        D, K = int(rng.choice([4, 6, 8])), int(rng.integers(2, 5))
        lean, streamed, sms = int(rng.integers(0, 2)), int(rng.integers(0, 2)), int(rng.choice([16, 132, 148]))
        kernel, S = _dispatch(F, T, D, K, lean, streamed, sms)
        nchunks = ((T + 31) // 32 * 32 + 127) // 128
        assert 1 <= S <= max(1, nchunks) and S in (1, 2, 4)
        if kernel == 1:
            assert D == 8 and lean and not streamed and F * S <= 2 * sms and -(-nchunks // S) <= 3
        elif kernel == 0:
            assert D == 8 and lean
        else:
            assert kernel == 2 and (D != 8 or not lean)
    k, s_ = ctypes.c_int(), ctypes.c_int()
    assert lib.pbb_em_dispatch(0, 10, 8, 3, 1, 0, 132, ctypes.byref(k), ctypes.byref(s_)) == -1
    assert lib.pbb_em_dispatch(5, 10, 5, 3, 1, 0, 132, ctypes.byref(k), ctypes.byref(s_)) == -3


def test_deferred_status_scope_host_logic():
    """_device.deferred_status / check_status with plain CPU tensors as status words: immediate raise outside a block,
    one read per word at the end of the block in call order, nesting, and no masking of an exception raised inside."""
    import torch
    from pb_bss_b200 import _device

    def raiser(tag):
        def on_error(s):
            raise ValueError(f'{tag}:{s}')
        return on_error

    ok, bad3, bad7 = torch.zeros(1, dtype=torch.int32), torch.tensor([3], dtype=torch.int32), torch.tensor([7], dtype=torch.int32)
    _device.check_status(ok, raiser('a'))                       # nothing to report
    with pytest.raises(ValueError, match='b:3'):
        _device.check_status(bad3, raiser('b'))                 # outside a block: on the spot
    seen = []
    with pytest.raises(ValueError, match='b:3'):               # the FIRST failing call of the block raises
        with _device.deferred_status() as scope:
            _device.check_status(ok, raiser('a'))
            _device.check_status(bad3, raiser('b'))
            _device.check_status(bad7, raiser('c'))
            seen.append(len(scope.items))
    assert seen == [3]
    with _device.deferred_status() as outer:                    # nested blocks: the inner one reports at its own end
        with pytest.raises(ValueError, match='c:7'):
            with _device.deferred_status():
                _device.check_status(bad7, raiser('c'))
        _device.check_status(ok, raiser('a'))
        assert len(outer.items) == 1
    with pytest.raises(KeyError):                               # an exception from the body is not replaced
        with _device.deferred_status():
            _device.check_status(bad3, raiser('b'))
            raise KeyError('body')
    _device.check_status(ok, raiser('a'))                       # and the scope is gone afterwards
    with pytest.raises(ValueError, match='b:3'):
        _device.check_status(bad3, raiser('b'))


def _header_code():
    text = open(os.path.join(ROOT, 'include', 'pbb.h')).read()
    return re.sub(r'/\*.*?\*/|//[^\n]*', ' ', text, flags=re.S)


def test_parsed_signatures():
    """Spot checks of the ctypes signatures _lib reads from include/pbb.h."""
    from pb_bss_b200 import _lib
    decls = _lib.parse_header()
    fit = decls['pbb_cacgmm_fit']
    assert len(fit.params) == 17 and fit.streamed
    assert fit.params[9].ctype is ctypes.POINTER(_lib.CacgmmOptions)
    assert [p.pointee for p in fit.params if p.name == 'eigenvalues'] == ['double']
    assert [p.pointee for p in fit.params if p.name == 'y'] == ['void']
    assert fit.params[4].ctype is ctypes.c_int and fit.params[4].pointee is None
    assert decls['pbb_cacgmm_workspace_bytes'].restype is ctypes.c_size_t
    assert decls['pbb_last_error'].restype is ctypes.c_char_p and decls['pbb_last_error'].params == ()
    assert decls['pbb_profile_reset'].restype is None
    assert decls['pbb_launch_count'].restype is ctypes.c_longlong
    host_only = {'pbb_last_error', 'pbb_version', 'pbb_launch_count', 'pbb_profile_enable', 'pbb_profile_reset',
                 'pbb_profile_dominant', 'pbb_profile_dump', 'pbb_streamed_task_order', 'pbb_em_dispatch',
                 'pbb_em_last_plan', 'pbb_stft_frames_per_cta', 'pbb_gammatone_chunk_length', 'pbb_srmr_fft_log2'}
    for name, decl in decls.items():
        names = [p.name for p in decl.params]
        if name in host_only or name.endswith(('_bytes', '_doubles')):
            assert not decl.streamed and 'stream' not in names, name
        else:  # every device entry point returns a status and takes the stream last
            assert decl.streamed and decl.restype is ctypes.c_int and names.count('stream') == 1, name
    assert sum(d.streamed for d in decls.values()) >= 100


def test_unknown_c_type_is_an_import_error(tmp_path):
    from pb_bss_b200 import _lib
    header = tmp_path / 'pbb.h'
    header.write_text('int pbb_ok(const double* x, long long n, void* stream);\n')
    assert _lib.parse_header(str(header))['pbb_ok'].params[1].ctype is ctypes.c_longlong
    for decl in ('int pbb_bad(float x, void* stream);', 'int pbb_bad(const double** x, void* stream);',
                 'unsigned pbb_bad(void);', 'double* pbb_bad(void);', 'int pbb_bad(int, void* stream);'):
        header.write_text(decl + '\n')
        with pytest.raises(ImportError, match='pbb_bad'):
            _lib.parse_header(str(header))


def test_mirrored_constants_match_the_header():
    """The integer constants and the three structs of _lib.py are hand-mirrored; they must equal include/pbb.h."""
    from pb_bss_b200 import _lib
    code = _header_code()
    consts = {n: int(v) for n, v in re.findall(r'#define\s+(PBB_\w+)\s+(-?\d+)\b', code)}
    for body in re.findall(r'\benum\s*\{(.*?)\}', code, flags=re.S):
        consts.update((n, int(v)) for n, v in re.findall(r'\b(PBB_\w+)\s*=\s*(-?\d+)', body))
    mirrored = {n: v for n, v in vars(_lib).items() if n.isupper() and type(v) is int}
    assert len(mirrored) >= 30
    for name, value in mirrored.items():
        c_name = name if name.startswith('PBB_') else 'PBB_' + name
        assert c_name in consts, f'_lib.{name} has no counterpart in include/pbb.h'
        assert value == consts[c_name], (name, value, consts[c_name])

    scalars = {'int': ctypes.c_int, 'double': ctypes.c_double, 'long long': ctypes.c_longlong}
    for c_name, cls in (('pbb_cacgmm_options', _lib.CacgmmOptions), ('pbb_mask_layout', _lib.MaskLayout),
                        ('pbb_nd_layout', _lib.NdLayout)):
        body = re.search(r'typedef\s+struct\s+%s\s*\{(.*?)\}\s*%s\s*;' % (c_name, c_name), code, flags=re.S).group(1)
        fields = []
        for ctype, name, dims in re.findall(r'([A-Za-z_][\w ]*?)\s+(\w+)\s*((?:\[\w+\])*)\s*;', body):
            t = scalars[' '.join(ctype.split())]
            for dim in reversed(re.findall(r'\[(\w+)\]', dims)):
                t = t * (int(dim) if dim.isdigit() else consts[dim])
            fields.append((name, t))
        assert cls._fields_ == fields, c_name
        assert ctypes.sizeof(cls) == sum(ctypes.sizeof(t) for _, t in fields), c_name  # no padding to disagree on


@pytest.fixture
def no_device_work(monkeypatch):
    """_device.call without a GPU: reading the stream fails the test, and the library function is replaced by a
    recorder, so a check that passed would be seen."""
    import torch
    from pb_bss_b200 import _device

    calls = []

    def stream():
        raise AssertionError('the stream was read')

    def stub(*args):
        calls.append(args)
        return 0
    monkeypatch.setattr(torch.cuda, 'current_stream', stream)
    for name in ('pbb_apply_mapping', 'pbb_mapping_from_score_matrix', 'pbb_cacgmm_fit'):
        monkeypatch.setitem(_device._entries, name, (stub,) + _device._entry(name)[1:])
    yield calls
    assert calls == []


def test_device_call_rejects_bad_arguments_before_any_device_work(no_device_work):
    import torch
    from pb_bss_b200 import _device
    f64 = torch.zeros(4, dtype=torch.float64)
    with pytest.raises(TypeError, match='not declared'):
        _device.call('pbb_no_such_function', None)
    with pytest.raises(TypeError, match='does not take a stream'):
        _device.call('pbb_cacgmm_workspace_bytes', 1, 1, 1, 1)
    with pytest.raises(TypeError, match='takes 6 arguments'):
        _device.call('pbb_apply_mapping', None, None, 1, 1, 1)
    with pytest.raises(TypeError, match='argument 1 wants torch.float64, got torch.float32'):
        _device.call('pbb_apply_mapping', torch.zeros(4, dtype=torch.float32), None, 1, 1, 1, None)
    with pytest.raises(TypeError, match='argument 6 wants torch.int32, got torch.int64'):
        _device.call('pbb_mapping_from_score_matrix', None, 1, 1, 0, None, torch.zeros(1, dtype=torch.int64))
    with pytest.raises(TypeError, match='argument 5 wants torch.int64, got torch.int32'):
        _device.call('pbb_mapping_from_score_matrix', None, 1, 1, 0, torch.zeros(1, dtype=torch.int32), None)
    with pytest.raises(ValueError, match='argument 1 is in pageable host memory'):
        _device.call('pbb_apply_mapping', f64, None, 1, 1, 1, None)
    with pytest.raises(TypeError, match='argument 2 is a pointer'):
        _device.call('pbb_apply_mapping', None, f64.data_ptr(), 1, 1, 1, None)
    with pytest.raises(TypeError, match='argument 3 is a scalar'):
        _device.call('pbb_apply_mapping', None, None, torch.tensor(1), 1, 1, None)
    with pytest.raises(TypeError, match='argument 10 wants no tensor'):
        _device.call('pbb_cacgmm_fit', None, 1, 1, 1, 4, 2, None, None, None, torch.zeros(1), None, None, None, None,
                     0, None)


def test_device_call_passes_null_ctypes_objects_and_the_stream(no_device_work, monkeypatch):
    import torch
    from pb_bss_b200 import _device, _lib

    class Stream:
        cuda_stream = 1234
    monkeypatch.setattr(torch.cuda, 'current_stream', lambda: Stream)
    opts = ctypes.byref(_lib.CacgmmOptions())
    _device.call('pbb_cacgmm_fit', None, 1, 1, 1, 4, 2, None, None, None, opts, None, None, None, None, 0, None)
    assert no_device_work == [(None, 1, 1, 1, 4, 2, None, None, None, opts, None, None, None, None, 0, None, 1234)]
    no_device_work.clear()
