"""NumPy / scipy restatement of the five trajnetplusplustools.metrics functions the reference's evaluator calls
(evaluator/trajnet_evaluator.py: average_l2, final_l2, collision, topk, nll).  TEST INFRASTRUCTURE.

The package that defines them upstream is not available here, so this module follows the definitions the scorer
documents (DESIGN.md section 2): ADE / FDE / the segment geometry of a collision / Top-k as in evaluator/eval_utils.py,
the KDE value of scipy.stats.gaussian_kde; the frame intersection of a collision and the skip / clip rules of the NLL are
restatements.  It is the CPU side of tests/golden/scoring_golden.npz (oracle/make_scoring_golden.py), where it stands in
for trajnetplusplustools.metrics under the reference's TrajnetEvaluator, and of scripts/score_bench.py.
Rows are anything with .frame, .x, .y (and .prediction_number for topk / nll).
"""
import numpy as np
from scipy.stats import gaussian_kde


def _xy(rows):
    return np.array([[r.x, r.y] for r in rows], dtype=np.float64).reshape(-1, 2)


def average_l2(path1, path2, n_predictions=12):
    assert len(path1) >= n_predictions
    assert len(path2) >= n_predictions
    d = _xy(path1[-n_predictions:]) - _xy(path2[-n_predictions:])
    return float(np.mean(np.linalg.norm(d, axis=-1)))


def final_l2(path1, path2):
    return float(np.linalg.norm(_xy(path1[-1:])[0] - _xy(path2[-1:])[0]))


def segments_collide(a, b, person_radius=0.1, inter_parts=2):
    """eval_utils.collision on two aligned [n, 2] arrays: 3 equally spaced points per segment, distance <= 2 r."""
    for i in range(len(a) - 1):
        pa = np.array((np.linspace(a[i][0], a[i + 1][0], inter_parts + 1), np.linspace(a[i][1], a[i + 1][1], inter_parts + 1)))
        pb = np.array((np.linspace(b[i][0], b[i + 1][0], inter_parts + 1), np.linspace(b[i][1], b[i + 1][1], inter_parts + 1)))
        if np.min(np.linalg.norm(pa - pb, axis=0)) <= 2 * person_radius:
            return True
    return False


def collision(path1, path2, n_predictions=12, person_radius=0.1, inter_parts=2):
    """Collision on the frames both tracks have within the last n_predictions rows of path1; none in common: False."""
    path1 = path1[-n_predictions:]
    common = {r.frame for r in path1} & {r.frame for r in path2}
    if not common:
        return False
    a = _xy([r for r in path1 if r.frame in common])
    b = _xy([r for r in path2 if r.frame in common])
    return segments_collide(a, b, person_radius, inter_parts)


def topk(primary_tracks, ground_truth, n_predictions=12, k_samples=3):
    """(smallest ADE, smallest FDE) over modes 0..k_samples-1, each minimum taken on its own (eval_utils.topk_ade /
    topk_fde)."""
    best_ade, best_fde = 1e10, 1e10
    for m in range(k_samples):
        mode = [t for t in primary_tracks if t.prediction_number == m]
        if not mode:
            continue
        a = average_l2(ground_truth, mode, n_predictions=n_predictions)
        f = final_l2(ground_truth, mode)
        if a < best_ade:
            best_ade = a
        if f < best_fde:
            best_fde = f
    return best_ade, best_fde


def kde_logpdf(samples, point):
    """log density at `point` [2] of scipy.stats.gaussian_kde over samples [K, 2]; None where scipy cannot fit it."""
    try:
        return float(gaussian_kde(np.asarray(samples, dtype=np.float64).T).logpdf(np.asarray(point, dtype=np.float64))[0])
    except (np.linalg.LinAlgError, ValueError):
        return None


def timestep_logpdf(samples, point, log_pdf_lower_bound=-20):
    """The clipped log-density of one timestep, or None where it is skipped: identical samples, no KDE, NaN, inf, > 100."""
    samples = np.asarray(samples, dtype=np.float64)
    if np.all(samples[1:] == samples[:-1]):
        return None
    lp = kde_logpdf(samples, point)
    if lp is None or np.isnan(lp):
        return None
    lp = max(lp, log_pdf_lower_bound)
    if np.isinf(lp) or lp > 100:
        return None
    return lp


def nll(primary_tracks, ground_truth, n_predictions=12, log_pdf_lower_bound=-20, n_samples=100):
    """-(mean over the kept timesteps of the clipped KDE log-density of the ground truth under all predicted modes)."""
    gt = _xy(ground_truth[-n_predictions:])
    frames = [t.frame for t in ground_truth][-n_predictions:]
    kept = []
    for t, frame in enumerate(frames):
        lp = timestep_logpdf(_xy([r for r in primary_tracks if r.frame == frame]), gt[t], log_pdf_lower_bound)
        if lp is not None:
            kept.append(lp)
    if not kept:
        raise Exception('All Predictions are Identical')
    return -(sum(kept) / len(kept))
