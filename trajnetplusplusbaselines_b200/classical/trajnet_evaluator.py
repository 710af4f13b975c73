"""`python -m trajnetplusplusbaselines_b200.classical.trajnet_evaluator --path <dataset> [--kf] [--sf] [--orca] [--cv]`:
the handcrafted baselines written file to file and scored (reference: classical/trajnet_evaluator.py).

Writes DATA_BLOCK/<dataset>/test_pred/{kf, sf, sf_opt, orca, orca_opt, cv}_modes<k>/<file>.ndjson in the reference's
order, skipping model folders that already exist, then scores them against test_private and prints the table unless
--write_only.  The scenes of a file go through the column pipeline in chunks (evaluator.evaluate_file with the batched
predictors of classical/batch.py) instead of one joblib task per scene; under torchrun the scenes are sharded over the
ranks.  Only mode 0 is predicted, like the reference's classical predict_scene.  The kf model averages 5 sampled
rollouts like the reference, drawn from torch's generator instead of NumPy's global RNG (DESIGN §8).
"""
import argparse
import os

from .. import evaluator


def model_list(args):
    """args.output as the reference builds it from the flags (classical/trajnet_evaluator.py:49-58)."""
    output = []
    if args.kf:
        output.append('/kf.pkl')
    if args.sf:
        output.extend(['/sf.pkl', '/sf_opt.pkl'])
    if args.orca:
        output.extend(['/orca.pkl', '/orca_opt.pkl'])
    if args.cv:
        output.append('/cv.pkl')
    return output


def parser():
    p = argparse.ArgumentParser()
    p.add_argument('--path', default='trajdata', help='directory of data to test')
    p.add_argument('--obs_length', default=9, type=int, help='observation length')
    p.add_argument('--pred_length', default=12, type=int, help='prediction length')
    p.add_argument('--write_only', action='store_true', help='write the predictions only, do not score them')
    p.add_argument('--disable-collision', action='store_true', help='disable collision metrics')
    p.add_argument('--labels', required=False, nargs='+', help='labels of models')
    p.add_argument('--normalize_scene', action='store_true', help='accepted and ignored, like the reference')
    p.add_argument('--modes', default=1, type=int, help='number of modes (the baselines write mode 0 only)')
    p.add_argument('--sf', action='store_true', help='consider socialforce in evaluation')
    p.add_argument('--orca', action='store_true', help='consider orca in evaluation')
    p.add_argument('--kf', action='store_true', help='consider kalman in evaluation')
    p.add_argument('--cv', action='store_true', help='consider constant velocity in evaluation')
    p.add_argument('--chunk', default=1024, type=int, help='scenes per batched call')
    return p


def main(argv=None, load_predictor=None):
    """Returns the scores ({label: {dataset: ...}}, scoring.trajnet_evaluate) or None with --write_only."""
    from .batch import load_predictor as batched
    args = parser().parse_args(argv)
    args.output = model_list(args)
    if not args.output:
        raise SystemExit('No handcrafted baseline mentioned: pass --kf, --sf, --orca and / or --cv')
    args.path = os.path.join('DATA_BLOCK', args.path, 'test_pred') + os.sep
    world = int(os.environ.get('WORLD_SIZE', '1'))
    if world > 1:                                            # torchrun: one process per GPU, scenes sharded over the ranks
        import torch
        import torch.distributed as dist
        if torch.cuda.is_available():
            torch.cuda.set_device(int(os.environ.get('LOCAL_RANK', '0')))
        dist.init_process_group('nccl' if torch.cuda.is_available() else 'gloo')
    try:
        written = evaluator.get_predictions(args, load_predictor=load_predictor or batched)
        if evaluator._rank_world()[0] != 0:
            return None
        for name, n in written.items():
            print('{}: {} scenes written'.format(name, n))
        if args.write_only:                                  # for submission to AICrowd
            print('Predictions written in test_pred folder')
            return None
        from ..scoring import trajnet_evaluate
        return trajnet_evaluate(args)
    finally:
        if world > 1:
            import torch.distributed as dist
            dist.destroy_process_group()


if __name__ == '__main__':
    main()
