"""Probe: how fast do kernels read pinned host memory directly (zero-copy over PCIe)?"""
import sys, time, ctypes
import numpy as np, torch
sys.path.insert(0, '.')
from oracle import synth
from pb_bss_b200 import _lib, _device
from pb_bss_b200.distribution import CACGMMTrainer

F, T, D, K, I = 513, 500, 8, 3, 100
y_pin = torch.from_numpy(synth.noise_stft(F, T, D)).pin_memory()
init_pin = torch.from_numpy(synth.init_affiliation(F, K, T)).pin_memory()
lib = _lib.load()
st = _device.stream_ptr()

def timed(fn, n=5):
    fn(); torch.cuda.synchronize()
    ts = []
    for _ in range(n):
        torch.cuda.synchronize(); t0 = time.perf_counter(); fn(); torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return min(ts) * 1e3

z = torch.empty(F, D, T, dtype=torch.complex128, device='cuda')
yd = y_pin.cuda()
def norm_dev():
    _lib.check(lib.pbb_normalize_observation(yd.data_ptr(), z.data_ptr(), F, T, D, _lib.PBB_C128, 1, st), 'n')
def norm_host():
    _lib.check(lib.pbb_normalize_observation(y_pin.data_ptr(), z.data_ptr(), F, T, D, _lib.PBB_C128, 1, st), 'n')
def h2d():
    y_pin.cuda(non_blocking=True); init_pin.cuda(non_blocking=True)
print('normalize device-resident  %.3f ms' % timed(norm_dev))
ms = timed(norm_host)
print('normalize zero-copy        %.3f ms  -> %.1f GB/s over PCIe' % (ms, y_pin.numel() * 16 / ms / 1e6))
ms = timed(h2d)
print('cudaMemcpyAsync y + init   %.3f ms  -> %.1f GB/s' % (ms, (y_pin.numel() * 16 + init_pin.numel() * 8) / ms / 1e6))
tr = CACGMMTrainer()
def e2e():
    tr.fit(y_pin, initialization=init_pin, iterations=I)
def resident():
    tr.fit(yd, initialization=init_d, iterations=I)
init_d = init_pin.cuda()
print('fit resident               %.3f ms' % timed(resident))
print('fit e2e streamed upload    %.3f ms' % timed(e2e))
def e2e_copy():
    tr.fit(y_pin.cuda(non_blocking=True), initialization=init_pin.cuda(non_blocking=True), iterations=I)
print('fit e2e memcpy then fit    %.3f ms' % timed(e2e_copy))
