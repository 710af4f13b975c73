// The evaluator's per-track displacement errors, shared by every kernel that scores a forecast (metrics.cu, shapley.cu).
// A file that includes this compiles with -fmad=false (build.py): with contraction the squares and sums would round
// differently from numpy's and the scores would not be the evaluator's bits.
#pragma once
#include <math.h>

namespace tb2 {

// eval_utils.ade / fde of one predicted track against the ground truth gt [T]: pred(t) returns the float64 prediction
// at frame t.  ADE = mean over the T frames of the Euclidean distance, FDE = the last frame's; NaN propagates.
template <class Pred>
__device__ __forceinline__ void ade_fde(Pred pred, const double2* __restrict__ gt, int T, double& ade, double& fde) {
    double sum = 0.0, last = NAN;
    for (int t = 0; t < T; ++t) {
        const double2 p = pred(t);
        const double dx = p.x - gt[t].x, dy = p.y - gt[t].y;
        last = sqrt(dx * dx + dy * dy);
        sum += last;
    }
    ade = sum / T;
    fde = last;
}

}  // namespace tb2
