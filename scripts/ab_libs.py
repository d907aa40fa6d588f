"""A/B timing and bit check of the C2 fit for several builds of the library: python scripts/ab_libs.py lib1.so lib2.so ...

For every build (PBB_LIB; 'default' = the package's own library) it times the C2 fit (F = 513, em_ws_kernel), the
F = 65 fit of scripts/one_fit_small.py (em_sticky_kernel) and the C2 fit from pinned host memory (streamed upload),
saves the fitted eigenvectors, eigenvalues and weights of each, and reports whether they are byte-identical to those
of the first build.  The library picks each fit's kernel from the problem alone, so other kernels are compared
through other shapes, not through settings."""
import os, sys, subprocess, tempfile
SHAPES = {'C2': (513, False), 'F65': (65, False), 'C2pinned': (513, True)}  # bins, pinned; T = 500, D = 8, K = 3
if sys.argv[1] == 'child':
    import numpy as np, torch
    sys.path.insert(0, '.')
    from oracle import synth
    from pb_bss_b200.distribution import CACGMMTrainer
    T, D, K, I = 500, 8, 3, 100
    out, line = {}, os.environ.get('PBB_LIB', 'default')
    for name, (F, pinned) in SHAPES.items():
        y = torch.from_numpy(synth.noise_stft(F, T, D))
        init = torch.from_numpy(synth.init_affiliation(F, K, T))
        y, init = (y.pin_memory(), init.pin_memory()) if pinned else (y.cuda(), init.cuda())
        tr = CACGMMTrainer()
        for _ in range(3): tr.fit(y, initialization=init, iterations=I)
        ts = []
        for _ in range(10):
            torch.cuda.synchronize(); e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
            e0.record(); tr.fit(y, initialization=init, iterations=I); e1.record(); torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        ts.sort()
        m = tr.fit(y, initialization=init, iterations=I)
        for key, v in (('vec', m.cacg.covariance_eigenvectors), ('val', m.cacg.covariance_eigenvalues), ('w', m.weight)):
            out['%s_%s' % (name, key)] = v.cpu().numpy() if torch.is_tensor(v) else np.asarray(v)
        line += '  %s min %.3f median %.3f ms' % (name, ts[0], ts[len(ts) // 2])
    np.savez(sys.argv[2], **out)
    print(line, flush=True)
else:
    import numpy as np
    tmp = tempfile.mkdtemp(prefix='ab_libs_')
    first = None
    for i, lib in enumerate(sys.argv[1:]):
        e = dict(os.environ)
        if lib != 'default': e['PBB_LIB'] = lib
        path = os.path.join(tmp, '%d.npz' % i)
        r = subprocess.run(['timeout', '300', sys.executable, __file__, 'child', path], env=e)
        if r.returncode != 0 or not os.path.exists(path):
            print('%s: failed (exit %d)' % (lib, r.returncode), flush=True)
            continue
        res = dict(np.load(path))
        if first is None:
            first = (lib, res)
            continue
        ref = first[1]
        diff = sorted(k for k in res if res[k].dtype != ref[k].dtype or res[k].shape != ref[k].shape
                      or res[k].tobytes() != ref[k].tobytes())
        print('%s vs %s: %s' % (lib, first[0], 'byte-identical' if not diff else 'DIFFERENT: ' + ', '.join(diff)),
              flush=True)
