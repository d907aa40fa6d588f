"""GPU checks of InputMetrics / OutputMetrics (pb_bss_b200.evaluation.wrapper) and GriffinLim.evaluate: the numbers
the reference publishes for the test_wrapper_values.py scenario, a K_target = K_source + 1 case, the shapes of the
reference's test_wrapper.py, PESQ, key errors, disabled SI-SDR and CUDA in / CUDA out."""
import numpy as np
import pytest

from oracle import sxr_oracle as O
from oracle.make_golden_metrics import wrapper_images

pytestmark = pytest.mark.gpu

INPUT_KEYS = ('stoi', 'mir_eval_sdr', 'mir_eval_sir', 'mir_eval_sar', 'srmr', 'invasive_sdr', 'invasive_snr',
              'invasive_sir')
OUTPUT_KEYS = ('stoi', 'mir_eval_sdr', 'mir_eval_sir', 'mir_eval_sar', 'mir_eval_selection', 'srmr', 'invasive_sdr',
               'invasive_snr', 'invasive_sir')


def _cuda(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _scenario(golden):
    m, b, s = golden('metrics'), golden('bss_eval'), golden('stoi')
    image, noise = wrapper_images(b['input_source'], b['input_observation'], m['wrapper_taps'])
    return dict(source=b['input_source'], observation=b['input_observation'], image=image, noise=noise), m, b, s


def _input_metrics(ex, cuda=False):
    from pb_bss_b200.evaluation import InputMetrics
    f = _cuda if cuda else (lambda x: x)
    return InputMetrics(observation=f(ex['observation']), speech_source=f(ex['source']), speech_image=f(ex['image']),
                        noise_image=f(ex['noise']), sample_rate=8000)


def _output_metrics(ex, cuda=False, **kw):
    from pb_bss_b200.evaluation import OutputMetrics
    f = _cuda if cuda else (lambda x: x)
    img = ex['image'][..., 0, :]
    noise = ex['noise'][..., 0, :]
    contribution = np.array([[img[0], np.zeros_like(img[1])], [np.zeros_like(img[0]), img[1]]])
    return OutputMetrics(speech_prediction=f(img + noise), speech_source=f(ex['source']),
                         speech_contribution=f(contribution), noise_contribution=f(np.array([noise, noise])),
                         sample_rate=8000, **kw)


@pytest.mark.parametrize('cuda', [False, True])
def test_input_metrics_published_values(golden, cuda):
    ex, m, b, s = _scenario(golden)
    metrics = _input_metrics(ex, cuda)
    assert metrics.K_source == 2 and metrics.channels == 3
    d = metrics.as_dict()
    assert tuple(d) == INPUT_KEYS
    if cuda:
        assert all(v.is_cuda for v in d.values())
        d = {k: v.cpu().numpy() for k, v in d.items()}
    for key in ('sdr', 'sir', 'snr'):
        np.testing.assert_allclose(d['invasive_' + key], m['anchor_input_invasive_' + key],
                                   rtol=m[f'anchor_input_invasive_{key}_rtol'])
    for key in ('sdr', 'sir', 'sar'):
        np.testing.assert_allclose(d['mir_eval_' + key], b['input_' + key], rtol=b['input_rtol'])
    np.testing.assert_allclose(d['stoi'], s['input_stoi'], rtol=s['input_rtol'])
    np.testing.assert_allclose(d['srmr'], m['anchor_input_srmr'], rtol=m['anchor_input_srmr_rtol'])


@pytest.mark.parametrize('cuda', [False, True])
def test_output_metrics_published_values(golden, cuda):
    ex, m, b, s = _scenario(golden)
    metrics = _output_metrics(ex, cuda)
    assert metrics.K_source == 2
    d = metrics.as_dict()
    assert tuple(d) == OUTPUT_KEYS
    if cuda:
        assert all(v.is_cuda for v in d.values())
        d = {k: v.cpu().numpy() for k, v in d.items()}
    for key in ('sdr', 'sir', 'snr'):
        np.testing.assert_allclose(d['invasive_' + key], m['anchor_output_invasive_' + key],
                                   rtol=m[f'anchor_output_invasive_{key}_rtol'])
    assert np.all(d['invasive_sir'] == np.inf)
    for key in ('sdr', 'sir', 'sar'):
        np.testing.assert_allclose(d['mir_eval_' + key], b['output_' + key], rtol=b['output_rtol'])
    np.testing.assert_array_equal(d['mir_eval_selection'], b['output_selection'])
    np.testing.assert_allclose(d['stoi'], s['output_stoi'], rtol=s['output_rtol'])
    np.testing.assert_allclose(d['srmr'], m['anchor_output_srmr'], rtol=m['anchor_output_srmr_rtol'])


def test_output_metrics_with_a_noise_estimate():
    """K_target = K_source + 1: speech estimates plus a noise estimate, the outputs in another order than the sources."""
    from pb_bss_b200.evaluation import OutputMetrics
    rng = np.random.default_rng(7)
    K, T = 2, 16000
    source = rng.standard_normal((K, T))
    mixing = np.array([[0.1, 1.0, 0.05], [0.9, 0.02, 0.1]])     # source k mostly on output 1 - k
    contribution = source[:, None, :] * mixing[:, :, None] + 0.01 * rng.standard_normal((K, K + 1, T))
    noise = 0.05 * rng.standard_normal((K + 1, T))
    noise[2] *= 20
    prediction = contribution.sum(0) + noise
    metrics = OutputMetrics(prediction, source, contribution, noise, sample_rate=8000, enable_si_sdr=True)
    d = metrics.as_dict()
    np.testing.assert_array_equal(d['mir_eval_selection'], [1, 0])
    selected = metrics.speech_prediction_selection
    np.testing.assert_array_equal(selected, prediction[[1, 0]])
    sdr, sir, snr, _ = O.output_sxr(contribution[:, [1, 0]], noise[[1, 0]], average_sources=False)
    for key, want in zip(('sdr', 'sir', 'snr'), (sdr, sir, snr)):
        np.testing.assert_allclose(d['invasive_' + key], want, rtol=1e-12)
    np.testing.assert_allclose(d['si_sdr'], O.si_sdr(source, prediction[[1, 0]]), rtol=1e-12)


def test_reference_shapes():
    """The shape checks of the reference's tests/test_evaluation/test_wrapper.py."""
    from pb_bss_b200.evaluation import InputMetrics, OutputMetrics
    rng = np.random.default_rng(8)
    channels, speakers, samples = 6, 2, 8000
    s = rng.normal(size=(speakers, samples))
    x = rng.normal(size=(speakers, channels, samples))
    n = rng.normal(size=(channels, samples))
    y = rng.normal(size=(channels, samples))
    contribution = rng.normal(size=(speakers, speakers + 1, samples))
    noise_contribution = rng.normal(size=(speakers + 1, samples))
    z = contribution.sum(0) + noise_contribution
    im = InputMetrics(observation=y, speech_source=s, speech_image=x, noise_image=n, sample_rate=8000,
                      enable_si_sdr=True)
    om = OutputMetrics(speech_prediction=z, speech_source=s, speech_contribution=contribution,
                       noise_contribution=noise_contribution, sample_rate=8000, enable_si_sdr=True)
    for m in im.mir_eval.values():
        assert m.shape == (speakers, channels)
    for m in im.invasive_sxr.values():
        assert m.shape == (speakers, channels)
    assert im.stoi.shape == (speakers, channels)
    assert im.si_sdr.shape == (speakers, channels)
    np.testing.assert_allclose(im.si_sdr, O.si_sdr(s[:, None], y[None]), rtol=1e-12)
    assert im.srmr.shape == (channels,)
    for m in om.mir_eval.values():
        assert m.shape == (speakers,)
    for m in om.invasive_sxr.values():
        assert m.shape == (speakers,)
    assert om.stoi.shape == (speakers,)
    assert om.si_sdr.shape == (speakers,)
    assert om.srmr.shape == (speakers,)
    for metrics in (im, om):
        with pytest.raises(NotImplementedError, match='P.862'):
            metrics.pesq
        with pytest.raises(NotImplementedError):
            metrics['pesq']
        assert 'pesq' not in metrics.as_dict() and 'pesq' in metrics._disabled_metric_names()


def test_key_errors_and_disabled_si_sdr(golden):
    from pb_bss_b200.evaluation.wrapper import VerboseKeyError
    ex, *_ = _scenario(golden)
    metrics = _input_metrics(ex)
    with pytest.raises(VerboseKeyError) as e:
        metrics['mir_eval_sdrr']
    assert "Close matches: ['mir_eval_sdr'" in str(e.value) and 'Disabled:' in str(e.value)
    with pytest.raises(ValueError, match='enable_si_sdr=True'):
        metrics['si_sdr']
    with pytest.raises(ValueError, match='enable_si_sdr=True'):
        _output_metrics(ex).si_sdr
    from pb_bss_b200.evaluation import OutputMetrics
    prediction = np.random.default_rng(10).standard_normal((2, 100))
    with pytest.raises(AssertionError, match='deviation'):
        OutputMetrics(prediction, np.ones((2, 100)), np.zeros((2, 2, 100)), np.zeros((2, 100)))
    with pytest.raises(AssertionError, match='deviation'):
        OutputMetrics(_cuda(prediction), _cuda(np.ones((2, 100))), _cuda(np.zeros((2, 2, 100))),
                      _cuda(np.zeros((2, 100))))
    OutputMetrics(prediction, np.ones((2, 100)), np.array([prediction, np.zeros((2, 100))]), np.zeros((2, 100)))


@pytest.mark.parametrize('cuda', [False, True])
def test_griffin_lim_evaluate(cuda):
    from oracle import transform_oracle as TO
    from pb_bss_b200.evaluation import mir_eval_sources
    from pb_bss_b200.transform import GriffinLim
    rng = np.random.default_rng(9)
    source = rng.standard_normal((2, 4032))       # istft(stft(x)) has this length again
    X = TO.stft(source, size=256, shift=64, fading=False)
    X = np.abs(X) * np.exp(1j * rng.uniform(-np.pi, np.pi, X.shape))
    gl = GriffinLim(_cuda(X) if cuda else X, size=256, shift=64)
    for _ in range(3):
        gl.step()
    got = gl.evaluate(_cuda(source) if cuda else source)
    if cuda:
        assert all(v.is_cuda for v in got.values())
        got = {k: float(v) for k, v in got.items()}
    x_hat = gl.x_hat.cpu().numpy() if cuda else gl.x_hat
    X_dash = gl.X_dash.cpu().numpy() if cuda else gl.X_dash
    sdr, sir, _, _ = mir_eval_sources(source, x_hat)
    np.testing.assert_allclose(got['mir_eval_sdr'], np.mean(sdr), rtol=1e-12)
    np.testing.assert_allclose(got['mir_eval_sir'], np.mean(sir), rtol=1e-12)
    D = X_dash - TO.stft(TO.istft(X_dash, size=256, shift=64, fading=False), size=256, shift=64, fading=False)
    np.testing.assert_allclose(got['inconsistency'], np.mean(D.real ** 2 + D.imag ** 2), rtol=1e-9)
