"""InputMetrics and OutputMetrics of pb_bss/evaluation/wrapper.py on the device: every metric of a separation result
through one object, with the reference's constructor arguments, input checks, lazily cached properties,
``as_dict()`` and ``metrics[name]``.

The inputs are copied to the device once.  OutputMetrics computes the mir_eval selection once, and every later metric
uses it (``speech_prediction[selection]`` and ``speech_contribution[:, selection]`` are device gathers).  ``as_dict()``
runs inside one ``deferred_status()`` block, so the status words of BSS Eval and STOI are read once, at the end.
NumPy in gives NumPy out; a CUDA tensor in gives CUDA tensors out.

Documented differences from the reference:
  - PESQ (ITU-T P.862) is not built: ``pesq`` raises NotImplementedError, it is listed among the disabled metrics,
    and ``as_dict()`` returns every other metric;
  - the metrics' own differences (module_mir_eval, module_stoi, module_srmr, module_si_sdr, sxr_module): integer and
    float32 input in fp64, and no NumPy RuntimeWarnings for zero powers.
"""
import difflib
import functools

import numpy as np
import torch

from .. import _device
from .module_mir_eval import mir_eval_sources
from .module_si_sdr import si_sdr
from .module_srmr import srmr
from .module_stoi import stoi
from .sxr_module import input_sxr, output_sxr

_PESQ = ('PESQ (ITU-T P.862) is not built in pb_bss_b200: there is no implementation of it on the device. The '
         'other metrics are available; as_dict() returns all of them.')
_SI_SDR_DISABLED = ('SI-SDR is disabled by default since it is only well-defined for non-reverberant single-channel '
                    'data. Enable it with `enable_si_sdr=True`.')


def _get_err_msg(msg, metrics):
    msg = f'{msg}'
    msg += '\nShapes: (is shape) (symbolic shape)'
    msg += f'\n\tspeech_prediction: {metrics.speech_prediction.shape} (K_target, N)'
    msg += f'\n\tspeech_source: {metrics.speech_source.shape} (K_source, N)'
    if metrics.speech_contribution is not None:
        msg += (f'\n\tspeech_contribution: '
                f'{metrics.speech_contribution.shape} (K_source, K_target, N)')
    if metrics.noise_contribution is not None:
        msg += (f'\n\tnoise_contribution: '
                f'{metrics.noise_contribution.shape} (K_target, N)')
    return msg


class VerboseKeyError(KeyError):
    """A KeyError whose message lists the available names by similarity to the unknown one (and what is disabled)."""

    def __str__(self):
        if len(self.args) in (2, 3):
            item, keys = self.args[:2]
            suggestions = difflib.get_close_matches(item, keys, cutoff=0, n=100)
            msg = f'{item!r}.\nClose matches: {suggestions!r}'
            if len(self.args) == 3:
                msg += f'\n{self.args[2]}'
            return msg
        return super().__str__()


def _metric(device_name):
    """A cached public metric: the device value of the attribute ``device_name``, as the caller gets it."""
    def get(self):
        return self._host(getattr(self, device_name))
    return functools.cached_property(get)


class _Metrics:
    """What InputMetrics and OutputMetrics share: NumPy / CUDA output, PESQ, SI-SDR gating, as_dict and lookup."""

    def _host(self, v):
        if isinstance(v, dict):
            return {k: self._host(x) for k, x in v.items()}
        if not self._numpy or not _device.is_tensor(v):
            return v
        v = v.cpu().numpy()
        return np.float64(v) if v.ndim == 0 else v

    @property
    def pesq(self):
        raise NotImplementedError(_PESQ)

    def _check_si_sdr(self):
        if not self.enable_si_sdr:
            raise ValueError(_SI_SDR_DISABLED)

    def _available_metric_names(self):
        names = list(self._METRICS)
        if self.enable_si_sdr:
            names.append('si_sdr')
        if self._has_invasive:
            names += ['invasive_sdr', 'invasive_snr', 'invasive_sir']
        return tuple(names)

    def _disabled_metric_names(self):
        disabled = ['pesq']
        if not self.enable_si_sdr:
            disabled.append('si_sdr')
        if not self._has_invasive:
            disabled += ['invasive_sdr', 'invasive_snr', 'invasive_sir']
        return disabled

    def as_dict(self):
        """Every available metric (the reference's keys without 'pesq'), in the reference's order."""
        names = self._available_metric_names()
        with _device.deferred_status():
            for name in names:
                getattr(self, '_d_' + name)
        return {name: self[name] for name in names}

    def __getitem__(self, item):
        assert isinstance(item, str), (type(item), item)
        try:
            return getattr(self, item)
        except AttributeError:
            pass
        raise VerboseKeyError(item, self._available_metric_names(), f'Disabled: {self._disabled_metric_names()}')

    mir_eval = _metric('_d_mir_eval')
    mir_eval_sdr = _metric('_d_mir_eval_sdr')
    mir_eval_sir = _metric('_d_mir_eval_sir')
    mir_eval_sar = _metric('_d_mir_eval_sar')
    invasive_sxr = _metric('_d_invasive_sxr')
    invasive_sdr = _metric('_d_invasive_sdr')
    invasive_sir = _metric('_d_invasive_sir')
    invasive_snr = _metric('_d_invasive_snr')
    stoi = _metric('_d_stoi')
    srmr = _metric('_d_srmr')
    si_sdr = _metric('_d_si_sdr')

    @functools.cached_property
    def _d_mir_eval_sdr(self):
        return self._d_mir_eval['sdr']

    @functools.cached_property
    def _d_mir_eval_sir(self):
        return self._d_mir_eval['sir']

    @functools.cached_property
    def _d_mir_eval_sar(self):
        return self._d_mir_eval['sar']

    @functools.cached_property
    def _d_invasive_sdr(self):
        return self._d_invasive_sxr['sdr']

    @functools.cached_property
    def _d_invasive_sir(self):
        return self._d_invasive_sxr['sir']

    @functools.cached_property
    def _d_invasive_snr(self):
        return self._d_invasive_sxr['snr']


def _dev(x):
    return None if x is None else _device.to_device(x)


class InputMetrics(_Metrics):
    """The metrics of the unprocessed observation (D, N) against the sources (K_source, N): per source and channel,
    or per channel for srmr.  The invasive SxR needs speech_image (K_source, D, N) and noise_image (D, N)."""

    _METRICS = ('stoi', 'mir_eval_sdr', 'mir_eval_sir', 'mir_eval_sar', 'srmr')

    def __init__(self, observation, speech_source, speech_image=None, noise_image=None, sample_rate: int = None,
                 enable_si_sdr: bool = False):
        """observation: when you pass D channels, you get D metrics per speaker; slice it to a singleton channel axis
        to select a reference channel.  enable_si_sdr: SI-SDR is only well defined for non-reverberant single-channel
        data, so it is disabled by default."""
        self.observation = observation
        self.speech_source = speech_source
        self.speech_image = speech_image
        self.noise_image = noise_image
        self.sample_rate = sample_rate
        self._has_image_signals = (speech_image is not None and noise_image is not None)
        self._has_invasive = self._has_image_signals
        self.samples = self.observation.shape[-1]
        self.channels = self.observation.shape[-2]
        self.K_source = self.speech_source.shape[0]
        self.enable_si_sdr = enable_si_sdr
        self.check_inputs()
        self._numpy = not any(_device.is_tensor(x) for x in (observation, speech_source, speech_image, noise_image))
        self._obs, self._src = _dev(observation), _dev(speech_source)

    def check_inputs(self):
        assert self.observation.ndim == 2, self.observation.shape
        assert self.speech_source.ndim == 2, self.speech_source.shape

    def _pairs(self):
        """reference (K_source, D, N) and estimation (K_source, D, N) as broadcast views: every channel's reference is
        the source, every source's estimate is the observation."""
        shape = (self.K_source, self.channels, self.samples)
        return self._src[:, None, :].expand(shape), self._obs[None].expand(shape)

    @functools.cached_property
    def _d_mir_eval(self):
        reference, estimation = self._pairs()
        return mir_eval_sources(reference=reference, estimation=estimation, return_dict=True,
                                compute_permutation=False)

    @functools.cached_property
    def _d_invasive_sxr(self):
        return input_sxr(_dev(self.speech_image), _dev(self.noise_image), average_sources=False,
                         average_channels=False, return_dict=True)

    @functools.cached_property
    def _d_stoi(self):
        return stoi(reference=self._src[:, None, :], estimation=self._obs[None], sample_rate=self.sample_rate)

    @functools.cached_property
    def _d_si_sdr(self):
        self._check_si_sdr()
        return si_sdr(reference=self._src[:, None, :], estimation=self._obs[None, :, :])

    @functools.cached_property
    def _d_srmr(self):
        return srmr(self._obs, self.sample_rate)


class OutputMetrics(_Metrics):
    """The metrics of a separation's output speech_prediction (K_target, N) against the sources speech_source
    (K_source, N), K_target = K_source or K_source + 1 (a noise estimate).  With compute_permutation the outputs are
    matched to the sources by mir_eval's SIR, and that selection is used by every metric.  The invasive SxR needs
    speech_contribution (K_source, K_target, N) and noise_contribution (K_target, N): the system's output for each
    source image and for the noise alone, which only a linear system has.  sample_rate is needed by stoi and srmr."""

    _METRICS = ('stoi', 'mir_eval_sdr', 'mir_eval_sir', 'mir_eval_sar', 'mir_eval_selection', 'srmr')

    def __init__(self, speech_prediction, speech_source, speech_contribution=None, noise_contribution=None,
                 sample_rate: int = None, enable_si_sdr: bool = False, compute_permutation: bool = True):
        self.speech_prediction = speech_prediction
        self.speech_source = speech_source
        self.speech_contribution = speech_contribution
        self.noise_contribution = noise_contribution
        self.sample_rate = sample_rate
        self._has_contribution_signals = (speech_contribution is not None and noise_contribution is not None)
        self._has_invasive = self._has_contribution_signals
        self.samples = self.speech_prediction.shape[-1]
        self.K_source = self.speech_source.shape[0]
        self.K_target = self.speech_prediction.shape[0]
        self.enable_si_sdr = enable_si_sdr
        self.compute_permutation = compute_permutation
        self._numpy = not any(_device.is_tensor(x) for x in (speech_prediction, speech_source, speech_contribution,
                                                            noise_contribution))
        self.check_inputs()
        self._pred, self._src = _dev(speech_prediction), _dev(speech_source)

    def _deviation(self):
        """np.std(np.abs(speech_prediction - sum of the contributions - noise_contribution)), computed eagerly: on the
        host for NumPy input, else on the device with one synchronisation."""
        if self._numpy:
            return np.std(np.abs(self.speech_prediction - np.sum(self.speech_contribution, axis=0)
                                 - self.noise_contribution))
        d = _dev(self.speech_prediction) - _dev(self.speech_contribution).sum(0) - _dev(self.noise_contribution)
        return float(d.abs().std(unbiased=False))

    def check_inputs(self):
        assert self.speech_prediction.ndim == 2, self.speech_prediction.shape
        assert self.speech_source.ndim == 2, self.speech_source.shape
        assert self.K_source <= 8, _get_err_msg(
            f'Number of source speakers (K_source) of speech_source is {self.K_source}. Expect a reasonable value '
            f'of 5 or less.', self)
        assert self.K_target <= 8, _get_err_msg(
            f'Number of target speakers (K_target) of speech_prediction is {self.K_target}. Expect a reasonable '
            f'value of 5 or less.', self)
        assert self.K_target in [self.K_source, self.K_source + 1], _get_err_msg(
            'Number of target speakers (K_target) should be equal to number of source speakers (K_source) or '
            'K_target + 1', self)
        assert self.speech_source.shape[1] == self.samples, _get_err_msg(
            'Num samples (N) of speech_source does not fit to theshape from speech_prediction', self)
        if self.speech_contribution is not None and self.noise_contribution is not None:
            K_source_, K_target_, samples_ = self.speech_contribution.shape
            assert self.samples == samples_, _get_err_msg(
                'Num samples (N) of speech_contribution does not fit to theshape from speech_prediction', self)
            assert self.K_target == K_target_, _get_err_msg(
                'Num target speakers (K_target) of speech_contribution does not fit to the shape from '
                'speech_prediction', self)
            assert self.K_source < 5, _get_err_msg(
                'Num source speakers (K_source) of speech_contribution does not fit to the shape from speech_source',
                self)
            K_target_, samples_ = self.noise_contribution.shape
            assert self.samples == samples_, _get_err_msg(
                'Num samples (N) of noise_contribution does not fit to the shape from speech_prediction', self)
            assert self.K_target == K_target_, _get_err_msg(
                'Num target speakers (K_target) of noise_contribution does not fit to the shape from '
                'speech_prediction', self)
            deviation = self._deviation()
            assert deviation < 1e-3, (
                'The deviation of speech prediction and the sum of individual contributions is expected to be low: '
                f'{deviation}')
        else:
            assert self.speech_contribution is None and self.noise_contribution is None, (
                'Expect that speech_contribution and noise_contribution are both None or given.\n'
                'Got:\n'
                f'speech_contribution: {self.speech_contribution}\n'
                f'noise_contribution: {self.noise_contribution}')

    mir_eval_selection = _metric('_d_mir_eval_selection')
    speech_prediction_selection = _metric('_d_speech_prediction_selection')

    @functools.cached_property
    def _d_mir_eval_selection(self):
        if self.compute_permutation:
            return self._d_mir_eval['selection']
        assert self.K_target == self.K_source, (self.K_target, self.K_source, self.compute_permutation)
        return torch.arange(self.K_source, device=self._pred.device)

    @functools.cached_property
    def _d_speech_prediction_selection(self):
        assert self.speech_prediction.ndim == 2, self.speech_prediction.shape
        assert self.speech_prediction.shape[0] < 10, self.speech_prediction.shape
        assert self.speech_prediction.shape[0] in (self.K_source, self.K_source + 1), self.speech_prediction.shape
        return self._pred.index_select(0, self._d_mir_eval_selection)

    @functools.cached_property
    def _d_mir_eval(self):
        return mir_eval_sources(reference=self._src, estimation=self._pred, return_dict=True,
                                compute_permutation=self.compute_permutation)

    @functools.cached_property
    def _d_invasive_sxr(self):
        selection = self._d_mir_eval_selection
        return output_sxr(_dev(self.speech_contribution).index_select(1, selection),
                          _dev(self.noise_contribution).index_select(0, selection), average_sources=False,
                          return_dict=True)

    @functools.cached_property
    def _d_stoi(self):
        return stoi(reference=self._src, estimation=self._d_speech_prediction_selection, sample_rate=self.sample_rate)

    @functools.cached_property
    def _d_srmr(self):
        return srmr(self._d_speech_prediction_selection, self.sample_rate)

    @functools.cached_property
    def _d_si_sdr(self):
        self._check_si_sdr()
        return si_sdr(reference=self._src, estimation=self._d_speech_prediction_selection)
