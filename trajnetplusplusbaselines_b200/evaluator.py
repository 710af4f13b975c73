"""Batched evaluator path (SURVEY.md 8f rank 1): what lstm/trajnet_evaluator.py:15-61 and
evaluator/write_utils.py do around the predictor -- read the test scenes of an ndjson file,
preprocess_test, predict, write_predictions -- with the per-scene joblib fan-out
(`Parallel(n_jobs=12)(delayed(predict_scene)...)`, trajnet_evaluator.py:61) replaced by chunks of
scenes going through ONE batched forward each (LSTMPredictor.predict_batch).

Multi-GPU (SURVEY.md 8e: scenes are independent, no data-path collective): under `torchrun` every rank takes a contiguous
range of the file's scenes (balanced by sum N^2, parallel.shard_scenes), writes its records to `<outfile>.part<rank>`, and
rank 0 concatenates the parts in rank order after a barrier -- the file is byte-identical to the single-process one.
"""
import inspect
import os
import shutil

from .data import (check_goal_ids, goal_file, load_goal_file, load_test_scenes_xy, paths_to_xy, preprocess_test,
                   read_ndjson_scenes, scene_goals, write_predictions, write_predictions_xy)


def load_test_scenes(filename, obs_length=9):
    """[(filename, scene_id, paths)] like evaluator/write_utils.load_test_datasets, already through
    preprocess_test (tracks that start after the observation period are dropped).

    Deliberate deviation in the written neighbour ids: the reference keeps the UN-preprocessed paths for
    write_predictions (lstm/trajnet_evaluator.py:57-64) while predict_scene drops the late tracks (:15-17), so the
    n-th predicted neighbour is labelled with the id of the n-th neighbour of the full scene
    (evaluator/write_utils.py:51-53,74-79) -- shifted whenever a dropped track precedes a kept one.  Here the ids
    come from the same preprocessed paths the predictions were made from, i.e. every trajectory carries its own id;
    primary rows, frames and scene rows are identical, and files without late tracks are identical throughout."""
    name = os.path.basename(filename)
    return [(name, scene_id, preprocess_test(paths, obs_length)) for scene_id, paths in read_ndjson_scenes(filename)]


def _takes_modes(predictor):
    fn = getattr(predictor, 'predict_batch_xy', None)
    if fn is None:
        return False
    try:
        return 'modes' in inspect.signature(fn).parameters
    except (TypeError, ValueError):
        return False


def batches_modes(predictor):
    """True for a predictor whose predict_batch_xy takes `modes` (S-GAN / VAE: every mode of every scene of a chunk in
    one batched decode, multimodal.py) and can decode its model that way."""
    supported = getattr(predictor, 'batch_decode_supported', None)
    return _takes_modes(predictor) and (supported is None or bool(supported()))


def _predict_xy(predictor, xys, pred_length, obs_length, modes, args, goals=None):
    if batches_modes(predictor):
        return predictor.predict_batch_xy(xys, n_predict=pred_length, obs_length=obs_length, args=args, modes=modes)
    if goals is not None:
        return predictor.predict_batch_xy(xys, goals, n_predict=pred_length, obs_length=obs_length, args=args)
    return predictor.predict_batch_xy(xys, n_predict=pred_length, obs_length=obs_length, args=args)


def predict_scenes(predictor, scenes, obs_length=9, pred_length=12, modes=1, chunk=1024, args=None, goals=None):
    """Predictions for a list of (filename, scene_id, paths), in order.  A predictor with
    predict_batch (LSTMPredictor) gets `chunk` scenes per forward at modes 1, one whose predict_batch_xy takes `modes`
    (S-GAN / VAE) `chunk` scenes per decode of all modes; any other predictor of the reference's call signature
    (classical, LSTM at modes > 1) is called scene by scene.  goals: per scene the goals [N, 2] of its tracks (a
    goal-conditioned model), else None (the predictor gets zeros, like the reference's)."""
    out = []
    if batches_modes(predictor):
        for i in range(0, len(scenes), chunk):
            xys = [paths_to_xy(paths) for _, _, paths in scenes[i:i + chunk]]
            out.extend(_predict_xy(predictor, xys, pred_length, obs_length, modes, args))
        return out
    if hasattr(predictor, 'predict_batch') and modes == 1:
        for i in range(0, len(scenes), chunk):
            part = [paths for _, _, paths in scenes[i:i + chunk]]
            if goals is not None:
                out.extend(predictor.predict_batch(part, goals[i:i + chunk], n_predict=pred_length, obs_length=obs_length,
                                                   args=args))
            else:
                out.extend(predictor.predict_batch(part, n_predict=pred_length, obs_length=obs_length, args=args))
        return out
    import numpy as np
    for i, (_, _, paths) in enumerate(scenes):
        goal = goals[i] if goals is not None else np.zeros((len(paths), 2))
        out.append(predictor(paths, goal, n_predict=pred_length, obs_length=obs_length, modes=modes, args=args))
    return out


def _rank_world(rank=None, world_size=None):
    """(rank, world_size): explicit arguments, else the initialised torch.distributed group, else (0, 1)."""
    if rank is not None and world_size is not None:
        return int(rank), int(world_size)
    try:
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized():
            return dist.get_rank(), dist.get_world_size()
    except ImportError:
        pass
    return 0, 1


def _barrier():
    try:
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            dist.barrier()
    except ImportError:
        pass


def _column_pipeline(predictor, modes):
    """The column pipeline (data.load_test_scenes_xy -> predict_batch_xy -> data.write_predictions_xy: native text passes,
    no Python object per track row) serves predictors that take arrays: at any `modes` when predict_batch_xy takes them
    (S-GAN / VAE), else at modes 1.  It writes the same bytes as the row pipeline."""
    if batches_modes(predictor):
        return True
    return hasattr(predictor, 'predict_batch_xy') and modes == 1 and not _takes_modes(predictor)


def evaluate_file(predictor, infile, outfile, obs_length=9, pred_length=12, modes=1, chunk=1024, args=None,
                  rank=None, world_size=None, goals=None, goals_path='goal file'):
    """ndjson in -> ndjson out (the records evaluator/write_utils.write_predictions appends).
    Returns the number of scenes of the file.  With world_size > 1 (arguments or the initialised process group) the
    scenes are sharded over the ranks; rank 0 assembles `outfile` from the per-rank parts.

    goals: for a goal-conditioned model the goals of the file (dict pedestrian id -> (x, y), read from goals_path).
    Every scene gets the goals of the tracks it keeps, in track order; a missing id raises before anything is written.
    Deliberate deviation: the reference passes the goals of the unfiltered scene, so a scene with a track that
    preprocess_test drops fails there on mismatched shapes."""
    columns = _column_pipeline(predictor, modes)
    if columns:
        scenes = load_test_scenes_xy(infile, obs_length)                 # [(xy, SceneMeta)]
        sizes = [xy.shape[1] for xy, _ in scenes]
        if goals is not None:
            goals = [scene_goals(goals, [meta.pedestrian] + list(meta.neigh_ids), goals_path) for _, meta in scenes]

        def run(part, part_goals, filename):
            preds = []
            for i in range(0, len(part), chunk):
                preds.extend(_predict_xy(predictor, [xy for xy, _ in part[i:i + chunk]], pred_length, obs_length, modes,
                                         args, None if part_goals is None else part_goals[i:i + chunk]))
            write_predictions_xy(preds, [meta for _, meta in part], filename, obs_length=obs_length, pred_length=pred_length)
    else:
        scenes = load_test_scenes(infile, obs_length)                    # [(filename, scene_id, paths)]
        sizes = [len(paths) for _, _, paths in scenes]
        if goals is not None:
            goals = [scene_goals(goals, [path[0].pedestrian for path in paths], goals_path) for _, _, paths in scenes]

        def run(part, part_goals, filename):
            preds = predict_scenes(predictor, part, obs_length, pred_length, modes, chunk, args, part_goals)
            write_predictions(preds, part, filename, obs_length=obs_length, pred_length=pred_length)
    rank, world = _rank_world(rank, world_size)
    if world == 1:
        if os.path.exists(outfile):
            os.remove(outfile)
        open(outfile, "w").close()
        if scenes:
            run(scenes, goals, outfile)
        return len(scenes)
    from .parallel import shard_scenes
    split = [0]
    for n in sizes:
        split.append(split[-1] + n)
    lo, hi = shard_scenes(split, world, rank)[:2]
    mine = scenes[lo:hi]
    part = "%s.part%d" % (outfile, rank)
    if os.path.exists(part):
        os.remove(part)
    open(part, "w").close()                                # an empty shard still leaves its (empty) part
    if mine:
        run(mine, None if goals is None else goals[lo:hi], part)
    _barrier()                                              # every part is complete
    if rank == 0:
        with open(outfile, "wb") as out:
            for r in range(world):
                with open("%s.part%d" % (outfile, r), "rb") as f:
                    shutil.copyfileobj(f, out)
        for r in range(world):
            os.remove("%s.part%d" % (outfile, r))
    _barrier()                                              # outfile is complete before any rank returns
    return len(scenes)


def prediction_folder(model, args):
    """Folder of a model's predictions under test_pred: `<model>_modes<k>`, or `<model>_sample_modes<k>` for the
    sampled predictions of args.sample (so that they never mix with the mean-trajectory files)."""
    sample = '_sample' if getattr(args, 'sample', False) else ''
    return os.path.basename(model).replace('.pkl', '') + sample + '_modes' + str(args.modes)


def _sampled_predictor(predictor):
    """--sample: the loaded LSTMPredictor's model in a SampledLSTMPredictor; any other predictor exits with a message."""
    from .lstm import LSTMPredictor
    if not isinstance(predictor, LSTMPredictor):
        raise SystemExit("--sample draws the modes of an LSTM model (LSTMPredictor); %s has no per-step normal to "
                         "sample: run it without --sample" % type(predictor).__name__)
    from .lstm.sampling import SampledLSTMPredictor
    try:
        return SampledLSTMPredictor(predictor.model)
    except NotImplementedError as e:
        raise SystemExit("--sample: %s" % e)


def get_predictions(args, load_predictor=None):
    """The write side of lstm/trajnet_evaluator.get_predictions (:28-64): for every model in args.output
    and every `*.ndjson` of the test folder, write `<path>/test_pred/<model>_modes<k>/<dataset>.ndjson`.
    With args.sample the predictor is a SampledLSTMPredictor of the loaded LSTM model (mode 0 the mean, the others drawn
    from the model's per-step normals) writing `<model>_sample_modes<k>`; a predictor that is not an LSTMPredictor exits
    with a message before anything is written.
    Existing model folders are skipped, like the reference does.  A goal-conditioned model (predictor.model.goal_flag)
    reads the goals of every test file from goal_files/test_private/<file>.pkl under the working directory, like the
    reference's evaluator.  Every goal file is loaded, and every pedestrian of every scene checked to have a goal, before
    the model folder is created: a missing file or id leaves nothing behind that a re-run would take for finished
    predictions.  Returns {model_name: scenes written}."""
    if load_predictor is None:
        def load_predictor(filename):
            from .lstm import LSTMPredictor
            predictor = LSTMPredictor.load(filename)
            predictor.model.to('cuda')
            return predictor
    rank = _rank_world()[0]
    pred_dir = args.path.rstrip(os.sep)       # .../test_pred -> the scenes are in .../test (trajnet_evaluator.py:31)
    test_dir = pred_dir[:-len('_pred')] if pred_dir.endswith('_pred') else pred_dir
    datasets = sorted(f for f in os.listdir(test_dir) if not f.startswith('.') and f.endswith('.ndjson'))
    written = {}
    for model in args.output:
        model_name = prediction_folder(model, args)
        out_dir = os.path.join(args.path, model_name)
        exists = os.path.exists(out_dir)
        _barrier()                                          # every rank has looked before rank 0 creates the folder
        if exists:
            if rank == 0:
                print('Predictions corresponding to {} already exist.'.format(model_name))
            continue
        predictor = load_predictor(model)
        if getattr(args, 'sample', False):
            predictor = _sampled_predictor(predictor)
        goals = {}
        if getattr(getattr(predictor, 'model', None), 'goal_flag', False):
            for dataset in datasets:
                goals[dataset] = load_goal_file(goal_file(dataset))
                check_goal_ids(goals[dataset], os.path.join(test_dir, dataset), goal_file(dataset))
        if rank == 0:
            os.makedirs(out_dir)
        _barrier()
        written[model_name] = sum(
            evaluate_file(predictor, os.path.join(test_dir, dataset), os.path.join(out_dir, dataset),
                          obs_length=args.obs_length, pred_length=args.pred_length, modes=args.modes,
                          chunk=args.chunk, args=args, goals=goals.get(dataset), goals_path=goal_file(dataset))
            for dataset in datasets)
    return written


def main(argv=None):
    """`python -m trajnetplusplusbaselines_b200.evaluator --path <dataset> --output model.pkl ...`: the
    prediction-writing half of `python -m trajnetbaselines.lstm.trajnet_evaluator` (same flags).  With --evaluate the
    files it writes are then scored against DATA_BLOCK/<dataset>/test_private (scoring.trajnet_evaluate, the metric half
    of the reference's evaluator) and the results table is printed."""
    import argparse
    parser = argparse.ArgumentParser()
    parser.add_argument('--path', default='trajdata', help='directory of data to test')
    parser.add_argument('--output', nargs='+', help='relative path to saved model')
    parser.add_argument('--obs_length', default=9, type=int)
    parser.add_argument('--pred_length', default=12, type=int)
    parser.add_argument('--normalize_scene', action='store_true')
    parser.add_argument('--modes', default=1, type=int)
    parser.add_argument('--chunk', default=1024, type=int, help='scenes per batched forward')
    parser.add_argument('--sample', action='store_true',
                        help='LSTM models: draw modes 1..k-1 from the per-step normals (mode 0 is the mean) into '
                             '<model>_sample_modes<k>')
    parser.add_argument('--evaluate', action='store_true',
                        help='after writing the predictions, score them against test_private and print the table')
    # the reference's scoring flags: they take effect with --evaluate (without it this tool only writes)
    parser.add_argument('--write_only', action='store_true', help='write the predictions only (the default without --evaluate)')
    parser.add_argument('--disable-collision', action='store_true', help='with --evaluate: do not score collisions')
    parser.add_argument('--labels', nargs='+', help='with --evaluate: model names in the table')
    args = parser.parse_args(argv)
    args.output = args.output if args.output is not None else []
    args.path = os.path.join('DATA_BLOCK', args.path, 'test_pred') + os.sep
    world = int(os.environ.get('WORLD_SIZE', '1'))
    if world > 1:                                            # torchrun: one process per GPU, scenes sharded over the ranks
        import torch
        import torch.distributed as dist
        if torch.cuda.is_available():
            torch.cuda.set_device(int(os.environ.get('LOCAL_RANK', '0')))
        dist.init_process_group('nccl' if torch.cuda.is_available() else 'gloo')
    written = get_predictions(args)
    if _rank_world()[0] == 0:
        for name, n in written.items():
            print('{}: {} scenes written'.format(name, n))
        if args.evaluate and not args.write_only:
            from .scoring import trajnet_evaluate
            trajnet_evaluate(args)
    if world > 1:
        import torch.distributed as dist
        dist.destroy_process_group()


if __name__ == '__main__':
    main()
