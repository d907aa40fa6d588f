"""Time per bin-iteration of the resident C2-shaped fit (T=500, D=8, K=3, 100 iterations) over the number of bins F,
for one or more builds of the library, alternated in one run:

  python scripts/l2_footprint_sweep.py [--rounds R] [--json OUT] lib1.so lib2.so ...   ('default' = the in-tree build)

The observation the fit re-reads every EM iteration grows with F.  While it fits the L2 the time per bin-iteration
stays flat; once it does not, the cyclic re-read misses and the time steps up.  The table lists the staged bytes
for a layout of 12 rows per ring stage (channels + repeated rows) and of 8 rows (channels only) next to each F.
F runs over whole multiples of the SM count (two CTAs per SM: every other point fills all CTA slots evenly).
Each fit is timed with CUDA events after an L2 flush (a 256 MiB buffer is overwritten), as bench.py does.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T, D, K, I = 500, 8, 3, 100


def staged_mb(F, rows):
    nchunks = ((T + 31) // 32 * 32 + 127) // 128
    return F * nchunks * rows * 128 * 16 / 1e6


def child(bins, reps):
    import torch
    sys.path.insert(0, ROOT)
    from oracle import synth
    from pb_bss_b200.distribution import CACGMMTrainer
    flush = torch.empty(256 << 20, dtype=torch.uint8, device='cuda')
    tr = CACGMMTrainer()
    out = {}
    for F in bins:
        y = torch.from_numpy(synth.noise_stft(F, T, D)).cuda()
        init = torch.from_numpy(synth.init_affiliation(F, K, T)).cuda()
        for _ in range(2):
            tr.fit(y, initialization=init, iterations=I)
        ts = []
        for _ in range(reps):
            flush.fill_(1)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            tr.fit(y, initialization=init, iterations=I)
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        ts.sort()
        out[F] = ts[len(ts) // 2]
    print(json.dumps(out), flush=True)


def gpu_info():
    import torch
    q = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.max.sm',
                        '--format=csv,noheader'], capture_output=True, text=True)
    return {'name': torch.cuda.get_device_name(0), 'nvidia_smi': q.stdout.strip(),
            'sms': torch.cuda.get_device_properties(0).multi_processor_count}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('libs', nargs='*')
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--reps', type=int, default=7)
    ap.add_argument('--multiples', default='2,3,4,5,6', help='F = m x SM count for these m')
    ap.add_argument('--json', help='write the results here')
    ap.add_argument('--child', help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        child([int(f) for f in args.child.split(',')], args.reps)
        return
    if not args.libs:
        ap.error('name at least one library')
    info = gpu_info()
    bins = [m * info['sms'] for m in map(int, args.multiples.split(','))]
    print(f"{info['name']} ({info['nvidia_smi']}), {info['sms']} SMs", flush=True)
    runs = {lib: [] for lib in args.libs}
    for r in range(args.rounds):
        for lib in args.libs:
            env = dict(os.environ)
            if lib != 'default':
                env['PBB_LIB'] = os.path.abspath(lib)
            p = subprocess.run([sys.executable, os.path.abspath(__file__), '--child', ','.join(map(str, bins)),
                                '--reps', str(args.reps)], env=env, capture_output=True, text=True, cwd=ROOT)
            if p.returncode != 0:
                sys.stderr.write(p.stdout + p.stderr)
                raise SystemExit(f'{lib}: child failed with exit code {p.returncode}')
            runs[lib].append({int(k): v for k, v in json.loads(p.stdout.strip().splitlines()[-1]).items()})
    print('ms per fit and ns per bin-iteration, min-max over the rounds: ' + ' | '.join(args.libs))
    print(f"{'F':>5} {'MB@12':>7} {'MB@8':>7}  " + '  '.join(f"{'ms/fit':>15} {'ns/bin-it':>13}" for _ in args.libs))
    table = []
    for F in bins:
        row = {'F': F, 'staged_mb_12_rows': staged_mb(F, 12), 'staged_mb_8_rows': staged_mb(F, 8)}
        cells = []
        for lib in args.libs:
            ms = sorted(run[F] for run in runs[lib])
            row[lib] = {'ms_per_fit': ms, 'ns_per_bin_iteration': [m * 1e6 / (F * I) for m in ms]}
            cells.append(f'{ms[0]:7.3f}-{ms[-1]:7.3f} {ms[0] * 1e6 / (F * I):6.2f}-{ms[-1] * 1e6 / (F * I):6.2f}')
        table.append(row)
        print(f'{F:5d} {row["staged_mb_12_rows"]:7.1f} {row["staged_mb_8_rows"]:7.1f}  ' + '  '.join(cells), flush=True)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, 'w') as f:
            json.dump({'gpu': info, 'shape': {'T': T, 'D': D, 'K': K, 'iterations': I}, 'rounds': args.rounds,
                       'reps_per_round': args.reps, 'rows': table}, f, indent=1)


if __name__ == '__main__':
    main()
