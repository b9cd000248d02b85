"""A/B of two source trees on one GPU: the parent commit's and this one's.

    python tools/ab_persistent.py --parent DIR --out DIR [--runs 3] [--no-build]

Builds both trees (make in sushi_b200/csrc), then runs `bench.py --no-cpu-baseline --no-load-leg` alternately from
each tree, `--runs` times each, on the default workload (config 3, uint8).  Afterwards each tree dumps its results
(`--dump-outputs`) on config 3 uint8, config 3 float32 and config 2, and the dumps are compared byte for byte.  The
card's name and power limit are read in the same process.  Writes OUT/ab.json and prints a summary: the headline
value, `kernel_ms_per_step` and the median SM clock of every run."""
import argparse
import filecmp
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip()


def bench(tree, extra):
    cmd = [sys.executable, os.path.join(tree, 'bench.py'), '--gpus', '1', '--no-cpu-baseline', '--no-load-leg'] + extra
    p = subprocess.run(cmd, cwd=tree, capture_output=True, text=True)
    if p.returncode != 0:
        raise RuntimeError('%s failed (%d):\n%s' % (' '.join(cmd), p.returncode, p.stderr[-4000:]))
    lines = [l for l in p.stdout.splitlines() if l.startswith('{')]
    return json.loads(lines[-1])


def summary(line):
    return {'value': line['value'], 'ms_per_step': line['ms_per_step'],
            'kernel_ms_per_step': line['roofline'].get('kernel_ms_per_step'), 'clocks': line.get('clocks')}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--parent', required=True, help='source tree of the parent commit')
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--no-build', action='store_true', help='both trees are built already')
    ap.add_argument('--out', required=True, help='directory for ab.json and the output dumps')
    args = ap.parse_args()
    trees = {'parent': os.path.abspath(args.parent), 'this': HERE}
    args.out = os.path.abspath(args.out)        # bench.py runs from each tree's directory
    os.makedirs(args.out, exist_ok=True)
    if not args.no_build:
        for t in trees.values():
            subprocess.check_call(['make', '-C', os.path.join(t, 'sushi_b200', 'csrc'), '-j8'], stdout=subprocess.DEVNULL)
    result = {'card': card(), 'runs': {k: [] for k in trees}, 'dumps': {}}
    for i in range(args.runs):
        for name, tree in trees.items():
            s = summary(bench(tree, []))
            result['runs'][name].append(s)
            print(name, i, json.dumps(s), flush=True)
    for label, extra in (('config3_u8', []), ('config3_f32', ['--sample-type', 'float32']),
                         ('config2_u8', ['--workload', 'config2', '--steps', '2', '--warmup', '1'])):
        if label.startswith('config3'):
            extra = extra + ['--steps', '2', '--warmup', '1']
        dirs = {}
        for name, tree in trees.items():
            dirs[name] = os.path.join(args.out, 'dump_%s_%s' % (label, name))
            bench(tree, extra + ['--dump-outputs', dirs[name]])
        same = all(filecmp.cmp(os.path.join(dirs['parent'], f), os.path.join(dirs['this'], f), shallow=False)
                   for f in ('diff.npy', 'time.npy'))
        result['dumps'][label] = 'identical' if same else 'DIFFERENT'
        print(label, result['dumps'][label], flush=True)
    result['card_after'] = card()
    with open(os.path.join(args.out, 'ab.json'), 'w') as f:
        json.dump(result, f, indent=1)
    vals = {k: [r['value'] for r in v] for k, v in result['runs'].items()}
    print('card:', result['card'])
    if not args.runs:
        return
    print('values:', json.dumps(vals))
    print('min(this) / max(parent) = %.4f, mean ratio = %.4f' % (
        min(vals['this']) / max(vals['parent']), (sum(vals['this']) / len(vals['this'])) / (sum(vals['parent']) / len(vals['parent']))))


if __name__ == '__main__':
    main()
