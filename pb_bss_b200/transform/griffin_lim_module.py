"""Griffin-Lim and MISI phase reconstruction on the device, pb_bss/transform/griffin_lim_module.py:6-130.

The state (x_hat, X_dash, X_dash_dash) lives on the device; ``step()`` only enqueues kernels (one STFT pass that also
forms X_dash, one iSTFT) and never synchronises the host.  The attributes are numpy arrays, copied on access, when the
instance was built from numpy, and CUDA tensors otherwise.
"""
import numpy as np
import torch

from .. import _device
from .fourier import griffin_lim_stft, istft, stft


class GriffinLim:
    """Griffin and Lim, "Signal estimation from modified short-time Fourier transform", IEEE TASSP 32(2), 1984.

    X: (K, T, F) target spectra, y: (num_samples,) mixture, first_guess: 'istft' (istft(X)) or 'y' (y / K for every
    k).  The transforms are stft / istft of this package with size, shift and fading and the other defaults."""

    def __init__(self, X, y=None, first_guess='istft', size=512, shift=128, fading=False):
        self._numpy = not _device.is_tensor(X)
        self.size, self.shift, self.fading = size, shift, fading
        self.X = X
        self.y = y
        self._X = _device.to_device(X, torch.complex128)
        assert self._X.dim() == 3, f'X: (K, T, F), got {tuple(self._X.shape)}'
        self._y = None if y is None else _device.to_device(y, torch.float64)
        self._X_dash_dash = self._X_dash = self._X
        if first_guess == 'istft':
            self._x_hat = self._istft(self._X)
        elif first_guess == 'white_gaussian_noise':
            # the reference's np.random.randn(size=...) raises this TypeError
            self._x_hat = np.random.randn(size=tuple(self._istft(self._X).shape))
        elif first_guess == 'y':
            K = self._X.shape[0]
            # text below [Gunawan2010MISI] equation 5.  K as a device tensor: torch turns the division by a host
            # scalar into a multiplication by its reciprocal, which is not NumPy's y / K
            K_dev = torch.full((), K, dtype=torch.float64, device=self._y.device)
            self._x_hat = (self._y[None, :] / K_dev).repeat(K, 1)
        else:
            raise ValueError(first_guess)

    def evaluate(self, speech_source):
        """dict of mir_eval_sdr and mir_eval_sir, the means over the sources of OutputMetrics(x_hat, speech_source,
        enable_si_sdr=True).mir_eval, and inconsistency, the mean of |X_dash - stft(istft(X_dash))|^2 with this
        instance's transforms.  np.float64 values for an instance built from numpy, 0-d CUDA tensors otherwise."""
        from ..evaluation import OutputMetrics
        from ..evaluation.sxr_module import get_variance_for_zero_mean_signal
        metrics = OutputMetrics(speech_prediction=self._x_hat, speech_source=_device.to_device(speech_source),
                                enable_si_sdr=True)
        inconsistency = get_variance_for_zero_mean_signal(
            self._X_dash - stft(self._istft(self._X_dash), size=self.size, shift=self.shift, fading=self.fading))
        sdr, sir = metrics.mir_eval['sdr'], metrics.mir_eval['sir']
        if self._numpy:
            return dict(mir_eval_sdr=np.mean(sdr.cpu().numpy()), mir_eval_sir=np.mean(sir.cpu().numpy()),
                        inconsistency=np.float64(inconsistency.cpu().numpy()))
        return dict(mir_eval_sdr=sdr.mean(), mir_eval_sir=sir.mean(), inconsistency=inconsistency)

    def _istft(self, X):
        return istft(X, size=self.size, shift=self.shift, fading=self.fading)

    def _out(self, t):
        return _device.to_host(t, self._numpy)

    @property
    def x_hat(self):
        return self._out(self._x_hat)

    @property
    def X_dash(self):
        return self._out(self._X_dash)

    @property
    def X_dash_dash(self):
        return self._out(self._X_dash_dash)

    def _step(self, y):
        self._X_dash_dash, self._X_dash = griffin_lim_stft(self._x_hat, self._X, y, self.size, self.shift,
                                                           self.fading)
        self._x_hat = self._istft(self._X_dash)

    def step(self):
        """X_dash_dash = stft(x_hat), X_dash = |X| exp(i angle(X_dash_dash)), x_hat = istft(X_dash)."""
        self._step(None)


class MISI(GriffinLim):
    """Gunawan and Sen, "Iterative phase estimation for the synthesis of separated sources from single-channel
    mixtures", IEEE SPL 17(5), 2010: the Griffin-Lim step on x_hat + (y - sum_k x_hat) / K."""

    def step(self):
        """Equations 5, 4, 3 and 2 of [Gunawan2010MISI] in one STFT pass and one iSTFT."""
        if self._y is None:
            raise TypeError("unsupported operand type(s) for -: 'NoneType' and 'ndarray'")
        if self._y.dim() != 1 or self._y.shape[0] != self._x_hat.shape[-1]:
            raise ValueError(f'operands could not be broadcast together with shapes {tuple(self._y.shape)} '
                             f'{tuple(self._x_hat.shape)}')
        self._step(self._y)
