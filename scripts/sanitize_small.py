"""Small fits for compute-sanitizer (memcheck / racecheck): lean + full persistent variants, CWMM, generic."""
import sys
import numpy as np
sys.path.insert(0, '.')
from oracle import synth
from pb_bss_b200.distribution import CACGMMTrainer, CWMMTrainer
y, _ = synth.structured_stft(12, 300, 8, 3, seed=1); init = synth.init_affiliation(12, 3, 300)
m = CACGMMTrainer().fit(y, initialization=init, iterations=4); m.predict(y)   # few bins: em_sticky_kernel (clusters)
yw, _ = synth.structured_stft(12, 2000, 8, 3, seed=5); iw = synth.init_affiliation(12, 3, 2000)
CACGMMTrainer().fit(yw, initialization=iw, iterations=3)   # 16 ring stages per bin: the task kernel em_ws_kernel
sal = np.random.RandomState(0).uniform(0.2, 1, size=(12, 300))
CACGMMTrainer().fit(y, initialization=init, iterations=3, saliency=sal)
y6, _ = synth.structured_stft(7, 260, 6, 4, seed=2); i6 = synth.init_affiliation(7, 4, 260)
CWMMTrainer().fit(y6, initialization=i6, iterations=3)
y3, _ = synth.structured_stft(3, 70, 3, 2, seed=3); i3 = synth.init_affiliation(3, 2, 70)
CACGMMTrainer().fit(y3, initialization=i3, iterations=3)
# streamed upload from pinned host memory (loader kernel + explicit task order) and K = 2 / 4 variants of the ws kernel
import torch
yp, ip = torch.from_numpy(y).pin_memory(), torch.from_numpy(init).pin_memory()
CACGMMTrainer().fit(yp, initialization=ip, iterations=4)
for K in (2, 4):
    yk, _ = synth.structured_stft(9, 200, 8, K, seed=4); ik = synth.init_affiliation(9, K, 200)
    CACGMMTrainer().fit(yk, initialization=ik, iterations=3)
# DHTV alignment: thread-block-cluster kernel (DSMEM) on a small plan, and the grid-barrier kernel's input range
from pb_bss_b200.permutation_alignment import DHTVPermutationAlignment
y13, _ = synth.structured_stft(13, 120, 8, 3, seed=6); i13 = synth.init_affiliation(13, 3, 120)
mask = CACGMMTrainer().fit(y13, initialization=i13, iterations=3).predict(y13)  # (F, K, T) numpy
al = DHTVPermutationAlignment(stft_size=24, segment_start=3, segment_width=6, segment_shift=2, main_iterations=4, sub_iterations=2)
al.calculate_mapping(np.ascontiguousarray(mask.transpose(1, 0, 2)))
print('ok')
