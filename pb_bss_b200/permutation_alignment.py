"""Frequency permutation alignment on the device, API of pb_bss/permutation_alignment.py.

``DHTVPermutationAlignment`` (segment-wise centroid matching, :133-355),
``GreedyPermutationAlignment`` (:592-714), ``OraclePermutationAlignment``
(:717-786) and ``apply_mapping`` (:54-104) run in CUDA (``pbb_dhtv_mapping``,
``pbb_score_matrix``, ``pbb_mapping_from_score_matrix``, ``pbb_chain_mapping``,
``pbb_apply_mapping``); the alignment plan is host logic.
"""
import ctypes

import numpy as np
import torch

from . import _device, _lib

__all__ = ['DHTVPermutationAlignment', 'GreedyPermutationAlignment',
           'OraclePermutationAlignment', 'apply_mapping', 'interleave',
           'sample_random_mapping']


def interleave(*lists):
    """Round-robin merge of lists of unequal length (:12-39)."""
    out = []
    for i in range(max((len(l) for l in lists), default=0)):
        for l in lists:
            if i < len(l):
                out.append(l[i])
    return iter(out)


def sample_random_mapping(K, F, random_state=np.random):
    """Random mapping (K, F) (:42-51)."""
    return np.stack([random_state.permutation(K) for _ in range(F)], axis=1)


def apply_mapping(mask, mapping):
    """mask (K, F, ...) , mapping (K, F) -> mask[mapping, range(F)] (:54-104)."""
    like_numpy = not _device.is_tensor(mask)
    m = _device.to_device(mask)
    out_dtype = m.dtype
    md = m.to(torch.float64)
    mp = _device.to_device(mapping).to(torch.int64).contiguous()
    K, F = mp.shape
    assert K < 20, (K, mp.shape)
    assert tuple(md.shape[:2]) == (K, F), (md.shape, mp.shape)
    T = int(np.prod(md.shape[2:])) if md.dim() > 2 else 1
    md = md.reshape(K, F, T).contiguous()
    out = _device.empty((K, F, T), torch.float64)
    _device.call('pbb_apply_mapping', md, mp, K, F, T, out)
    out = out.reshape(m.shape).to(out_dtype)
    return _device.to_host(out, like_numpy)


class _PermutationAlignment:
    def calculate_mapping(self, mask, *args, **kwargs):
        raise NotImplementedError()

    def __call__(self, mask, *args, **kwargs):
        """mask (K, F, T) -> aligned mask (:116-125)."""
        mapping = self.calculate_mapping(mask, *args, **kwargs)
        return self.apply_mapping(mask, mapping)

    @staticmethod
    def apply_mapping(mask, mapping):
        return apply_mapping(mask, mapping)


class DHTVPermutationAlignment(_PermutationAlignment):
    """Segment-wise frequency permutation alignment [TranVu2015BSS] (:133-355)."""

    def __init__(self, *, stft_size, segment_start, segment_width,
                 segment_shift, main_iterations, sub_iterations,
                 similarity_metric='cos', algorithm='greedy'):
        self.stft_size = stft_size
        self.segment_start = segment_start
        self.segment_width = segment_width
        self.segment_shift = segment_shift
        self.main_iterations = main_iterations
        self.sub_iterations = sub_iterations
        self.similarity_metric = similarity_metric
        self.algorithm = algorithm
        # like the reference (:157-162) an unknown metric fails here, an unknown algorithm when it is first used
        self._metric = _metric_code(similarity_metric)

    @classmethod
    def from_stft_size(cls, stft_size, similarity_metric='cos'):
        """Presets of the reference (:164-184)."""
        if stft_size == 512:
            start = 70
        elif stft_size == 1024:
            start = 100
        else:
            raise ValueError('There is no default for stft_size={}.', stft_size)
        return cls(stft_size=stft_size, segment_start=start, segment_width=100,
                   segment_shift=20, main_iterations=20, sub_iterations=2,
                   similarity_metric=similarity_metric)

    @property
    def alignment_plan(self):
        """List of [iterations, start, end] (:204-293)."""
        F = self.stft_size // 2 + 1
        if self.segment_start + self.segment_width > F:
            raise ValueError(
                f'segment_start ({self.segment_start}) '
                f'+ segment_width ({self.segment_width})\n'
                f'must be smaller than stft_size // 2 + 1 ({F}),\n'
                f'but it is {self.segment_start + self.segment_width}')
        lower = [[self.sub_iterations, s, s + self.segment_width]
                 for s in range(self.segment_start + self.segment_shift,
                                F - self.segment_width, self.segment_shift)]
        higher = [[self.sub_iterations, s, s + self.segment_width]
                  for s in range(self.segment_start - self.segment_shift, 0,
                                 -self.segment_shift)]
        first = [self.main_iterations, self.segment_start,
                 self.segment_start + self.segment_width]
        if lower:
            lower[-1][-1] = F
        else:
            first[-1] = F
        if higher:
            higher[-1][1] = 0
        else:
            first[1] = 0
        return [first] + list(interleave(lower, higher))

    def calculate_mapping(self, mask, plot=False):
        """mask (K, F, T) -> reverse mapping (K, F) int64 (:295-355)."""
        like_numpy = not _device.is_tensor(mask)
        m = _device.to_device(mask).to(torch.float64).contiguous()
        K, F, T = m.shape
        assert K < 10, (K, 'Sure?')
        assert F % 2 == 1, (F, 'Sure? Usually F is odd.')
        plan = np.asarray(self.alignment_plan, dtype=np.int32)
        assert plan[:, 2].max() <= F, (plan, F)
        plan = np.ascontiguousarray(plan)
        plan_p = plan.ctypes.data_as(ctypes.POINTER(ctypes.c_int))
        lib = _lib.load()
        feat = _device.empty((K, F, T), torch.float64)
        cent = _device.empty((int(lib.pbb_dhtv_scratch_doubles(K, T, plan_p, int(plan.shape[0]))),), torch.float64)
        mapping = _device.empty((K, F), torch.int64)
        if self.algorithm not in _ALGORITHMS:
            raise ValueError(self.algorithm)   # _mapping_from_score_matrix (:588-589)
        _device.call('pbb_dhtv_mapping_ex', m, K, F, T, plan_p, int(plan.shape[0]), feat, cent, mapping, self._metric,
                     _ALGORITHMS[self.algorithm])
        return _device.to_host(mapping, like_numpy)


_METRICS = {'multiply': 0, 'cos': 1, 'euclidean': 2}
_ALGORITHMS = {'greedy': 0, 'optimal': 1}


def _metric_code(similarity_metric):
    """_ScoreMatrix.from_name (:420-441): unknown names raise with the suggestions."""
    try:
        return _METRICS[similarity_metric]
    except (KeyError, TypeError):
        raise AttributeError(
            f"type object '_ScoreMatrix' has no attribute {similarity_metric!r}\n"
            'Suggestions: cos, euclidean, from_name, multiply') from None


def _score_matrix(mask, reference_mask, metric, F, source_strides=None):
    """(K, F, T) device masks -> scores (F, K, K) on the device (:380-420).

    ``source_strides`` = element strides between sources of (mask, reference)
    when they are views with F bins into larger arrays.
    """
    K, _, T = mask.shape
    ms, rs = source_strides or (mask.shape[1] * T, reference_mask.shape[1] * T)
    scores = _device.empty((F, K, K), torch.float64)
    _device.call('pbb_score_matrix', mask, reference_mask, ms, rs, K, F, T, metric, scores)
    return scores


def _mapping_from_score_matrix(score_matrix, algorithm='optimal'):
    """score_matrix (..., K, K) -> mapping (K, ...) (:458-590)."""
    like_numpy = not _device.is_tensor(score_matrix)
    sc = _device.to_device(np.asanyarray(score_matrix) if like_numpy else score_matrix).to(torch.float64)
    *F, K, K_ = sc.shape
    assert K == K_, (tuple(sc.shape), K, K_)
    if algorithm not in _ALGORITHMS:
        raise ValueError(algorithm)
    n = int(np.prod(F)) if F else 1
    sc = sc.reshape(n, K, K).contiguous()
    mapping = _device.empty((K, n), torch.int64)
    status = torch.zeros(1, dtype=torch.int32, device=sc.device)
    _device.call('pbb_mapping_from_score_matrix', sc, n, K, _ALGORITHMS[algorithm], mapping, status)
    def on_error(s):
        # message of scipy.optimize.linear_sum_assignment, like the reference (:511-513)
        raise ValueError('score matrix is infeasible')
    _device.check_status(status, on_error)
    return _device.to_host(mapping.reshape(K, *F), like_numpy)


class GreedyPermutationAlignment(_PermutationAlignment):
    """Align every bin to its lower neighbour, then chain the mappings (:592-714).

    As in the reference the pairwise assignment is always the greedy one; the
    ``algorithm`` argument is stored but not used (:702-703).
    """

    def __init__(self, similarity_metric='euclidean', algorithm='optimal'):
        try:
            self._metric = _metric_code(similarity_metric)
        except Exception:
            raise ValueError(similarity_metric)
        self.similarity_metric = similarity_metric
        self.algorithm = algorithm

    def calculate_mapping(self, mask):
        """mask (K, F, T) -> mapping (K, F) int64 (:612-714)."""
        like_numpy = not _device.is_tensor(mask)
        m = _device.to_device(mask).to(torch.float64).contiguous()
        K, F, T = m.shape
        assert K < 10, (K, 'Sure?')
        assert F % 2 == 1, (F, 'Sure? Usually F is odd.', tuple(m.shape))
        mapping = _device.empty((K, F), torch.int64)
        pair = None
        if F > 1:
            # scores between mask[:, 1:] and mask[:, :-1]: two views of the same array
            scores = _device.empty((F - 1, K, K), torch.float64)
            _device.call('pbb_score_matrix', m[:, 1:], m, F * T, F * T, K, F - 1, T, self._metric, scores)
            pair = _mapping_from_score_matrix(scores, 'greedy')
        _device.call('pbb_chain_mapping', pair, K, F, mapping)
        return _device.to_host(mapping, like_numpy)


class OraclePermutationAlignment(_PermutationAlignment):
    """Align every bin to a reference mask (:717-786)."""

    def __init__(self, similarity_metric='euclidean', algorithm='optimal'):
        assert algorithm in ['greedy', 'optimal'], algorithm
        self._metric = _metric_code(similarity_metric)
        self.similarity_metric = similarity_metric
        self.algorithm = algorithm

    def calculate_mapping(self, mask, reference_mask):
        """mask, reference_mask (K, F, T) -> mapping (K, F) int64 (:723-786)."""
        like_numpy = not _device.is_tensor(mask)
        m = _device.to_device(mask).to(torch.float64).contiguous()
        r = _device.to_device(reference_mask).to(torch.float64).contiguous()
        assert m.shape == r.shape, (tuple(m.shape), tuple(r.shape))
        K, *F, T = m.shape
        assert K < 10, (K, 'Sure?')
        if len(F) == 1:
            assert F[0] % 2 == 1, (F, 'Sure? Usually F is odd.', tuple(m.shape))
        n = int(np.prod(F)) if F else 1
        scores = _score_matrix(m.reshape(K, n, T), r.reshape(K, n, T), self._metric, n)
        mapping = _mapping_from_score_matrix(scores, self.algorithm)
        return _device.to_host(mapping.reshape(K, *F), like_numpy)
