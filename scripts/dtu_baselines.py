"""The paper's EMS / MBF baseline comparison on the ten DTU scans (the reference's scripts/ems_pproc.sh, mbf_pproc.sh,
ems_eval.sh and mbf_eval.sh) on the GPU, through dbw_b200.baselines:

    python scripts/dtu_baselines.py preprocess --reference <checkout> --out_dir <ems or mbf runs>/dtu --name ems --tag default_noground --filter_ground
    python scripts/dtu_baselines.py ems_eval --reference <checkout> --baseline_dir <ems runs>/dtu --dtu_dir <datasets>/DTU --out_dir <runs>/ems --tag default_noground
    python scripts/dtu_baselines.py mbf_eval --reference <checkout> --baseline_dir <mbf runs>/dtu --dtu_dir <datasets>/DTU --out_dir <runs>/mbf --tag default_noground

The scans are read by the reference's own DTUDataset (`--reference`: a checkout of monniert/differentiable-blocksworld whose
datasets are in place), with compat's stand-ins for its PyTorch3D imports; nothing else of the checkout is used.  Writes, under
<out_dir>/<tag>: {scan}_scale.npy and {scan}.ply (preprocess), or {scan}_scores.tsv and dtu_scores_{scan}.tsv (evaluations).
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

EVAL_SCAN_IDS = [f'scan{i}' for i in [24, 31, 40, 45, 55, 59, 63, 75, 83, 105]]


def datasets(reference):
    """tag -> the reference's DTUDataset(split='train', img_size=(300, 400), tag=tag), loaded lazily"""
    import dbw_b200.compat as compat
    compat.install()
    sys.path.insert(0, os.path.join(os.path.abspath(reference), 'src'))
    from dataset import get_dataset                                   # the reference's file

    class Lazy(dict):
        def items(self):
            for tag in EVAL_SCAN_IDS:
                yield tag, get_dataset('dtu')(split='train', img_size=(300, 400), tag=tag)
    return Lazy()


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument('command', choices=['preprocess', 'ems_eval', 'mbf_eval'])
    ap.add_argument('--reference', required=True, help='checkout of monniert/differentiable-blocksworld (for its DTUDataset)')
    ap.add_argument('--out_dir', required=True)
    ap.add_argument('-t', '--tag', required=True, help='Run tag of the experiment')
    ap.add_argument('-n', '--name', choices=['ems', 'mbf'], help='Name of the baseline model (preprocess)')
    ap.add_argument('-f', '--filter_ground', action='store_true', help='remove the RANSAC ground plane (preprocess)')
    ap.add_argument('-e', '--ems_tag', help='EMS tag of the experiment (ems_eval; default: --tag)')
    ap.add_argument('--mbf_tag', help='MBF tag of the experiment (mbf_eval; default: --tag)')
    ap.add_argument('--baseline_dir', help='directory holding <ems_tag or mbf_tag>/ with the fitted baseline (evaluations)')
    ap.add_argument('--dtu_dir', help='DTU directory with ObsMask/ and Points/stl/ (evaluations)')
    ap.add_argument('-s', '--seed', type=int, default=1234, help='Seed')
    args = ap.parse_args()
    assert args.tag != ''
    from dbw_b200 import baselines as B
    run_dir = os.path.join(args.out_dir, args.tag)
    if args.command == 'preprocess':
        if args.name is None:
            ap.error('preprocess needs --name')
        B.DTU3DPreprocess(run_dir, args.name, filter_ground=args.filter_ground).run(datasets(args.reference), seed=args.seed)
        return
    if args.baseline_dir is None or args.dtu_dir is None:
        ap.error(f'{args.command} needs --baseline_dir and --dtu_dir')
    ems = args.command == 'ems_eval'
    src = os.path.join(args.baseline_dir, (args.ems_tag if ems else args.mbf_tag) or args.tag)
    cls = B.EMSEvaluator if ems else B.MBFEvaluator
    scores = cls(run_dir, src).run(datasets(args.reference), args.dtu_dir, seed=args.seed)
    for tag, s in scores.items():
        print(tag, ', '.join(f'{k}={v:.5f}' for k, v in s.items()))


if __name__ == '__main__':
    main()
