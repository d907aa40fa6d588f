"""A/B of the DHTV alignment kernels: cluster / DSMEM kernel (default) vs grid-barrier kernel (PBB_DHTV_COOP=1) on
cACGMM masks, for every similarity metric and both assignments; time per calculate_mapping at C3 size.  The kernels add the centroid in different orders, so a mapping
may differ where a decision lies within rounding of a tie; tests/test_permutation_gpu.py checks them against the
oracle with that precondition."""
import os, subprocess, sys, tempfile
if len(sys.argv) > 1 and sys.argv[1] == 'child':
    import numpy as np, torch
    sys.path.insert(0, '.')
    from oracle import synth
    from pb_bss_b200.distribution import CACGMMTrainer
    from pb_bss_b200.permutation_alignment import DHTVPermutationAlignment
    out = {}
    for (F, T, K, seed) in ((513, 500, 3, 5), (257, 300, 2, 6), (513, 200, 4, 7)):
        y, _ = synth.structured_stft(F, T, 8, K, seed=seed)
        init = synth.init_affiliation(F, K, T, seed=7)
        m = CACGMMTrainer().fit(torch.from_numpy(y).cuda(), initialization=torch.from_numpy(init).cuda(), iterations=15)
        mask = m.predict(torch.from_numpy(y).cuda()).permute(1, 0, 2).contiguous()
        for metric in ('cos', 'multiply', 'euclidean'):
            for algorithm in ('greedy', 'optimal'):
                # the metric is fixed when the aligner is constructed: one aligner per metric
                al = DHTVPermutationAlignment(stft_size=2 * (F - 1), segment_start=100 if F == 513 else 70,
                                              segment_width=100, segment_shift=20, main_iterations=20,
                                              sub_iterations=2, similarity_metric=metric, algorithm=algorithm)
                out[f'{F}_{K}_{metric}_{algorithm}'] = al.calculate_mapping(mask).cpu().numpy()
        if F == 513 and K == 3:
            al = DHTVPermutationAlignment.from_stft_size(1024)
            for _ in range(3): al.calculate_mapping(mask)
            ts = []
            for _ in range(9):
                torch.cuda.synchronize(); e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
                e0.record(); al.calculate_mapping(mask); e1.record(); torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1))
            ts.sort()
            print(f'[{sys.argv[2]}] calculate_mapping F=513 T=500 K=3 cos: min {ts[0]:.3f} median {ts[4]:.3f} ms', flush=True)
    np.savez(sys.argv[3], **out)
else:
    import numpy as np
    res = {}
    tmp = tempfile.mkdtemp()
    for tag, env in (('cluster', {}), ('coop', {'PBB_DHTV_COOP': '1'})):
        e = dict(os.environ); e.update(env)
        path = os.path.join(tmp, f'ab_dhtv_{tag}.npz')
        subprocess.run(['timeout', '300', sys.executable, __file__, 'child', tag, path], env=e, check=True)
        res[tag] = np.load(path)
    for k in res['cluster'].files:
        same_coop = np.array_equal(res['cluster'][k], res['coop'][k])
        nonid = int((res['cluster'][k] != np.arange(res['cluster'][k].shape[0])[:, None]).any(0).sum())
        print(f'{k}: cluster == coop {same_coop}, bins with a non-identity mapping {nonid}')
    # the metrics really differ: not every metric gives the same mapping
    for F, K in ((513, 3), (257, 2), (513, 4)):
        maps = [res['cluster'][f'{F}_{K}_{m}_greedy'] for m in ('cos', 'multiply', 'euclidean')]
        print(f'F={F} K={K}: mappings of cos / multiply / euclidean pairwise equal: '
              f'{[bool(np.array_equal(a, b)) for a, b in ((maps[0], maps[1]), (maps[0], maps[2]), (maps[1], maps[2]))]}')
