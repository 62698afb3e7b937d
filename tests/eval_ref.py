"""A float64 NumPy restatement of p2pvg_metrics_fold (include/p2pvg_b200.h) and of evaluate_split's aggregation.

``fold_ref`` adds one batch's scores to the totals in the kernel's documented order: per bin its columns in column order,
each column's rows in row order, one Python float add (or multiply) per value, so that its totals are bit-identical to the
kernel's.  ``best_ref`` is the best-sample rule: the sample whose mean over the segment's frames (summed in frame order,
then divided) is best, the first on ties, the first NaN mean if there is one -- torch's argmax / argmin, which
metrics.best_of applies."""
import math

import numpy as np

N_SUMS, N_COUNTS = 3, 4


def new_totals(n_bins, nm):
    return dict(sums=np.zeros((n_bins, nm, N_SUMS)), counts=np.zeros((n_bins, nm, N_COUNTS), np.int64),
                rows=np.zeros(n_bins, np.int64))


def best_ref(v, higher):
    """v: [nsample][F] python floats of one row and metric -> the best sample's index."""
    best, bm = 0, None
    for s, vs in enumerate(v):
        acc = 0.0
        for a in vs:
            acc += a
        m = acc / len(vs)
        if s == 0:
            bm = m
        elif not math.isnan(bm) and (math.isnan(m) or (m > bm if higher else m < bm)):
            best, bm = s, m
    return best


def fold_ref(tot, scores, segs, col_bin, B, ns, higher_mask):
    """Adds one batch to tot (new_totals): scores float64 [n_pairs, nm]; segs [(first pair, first column, F)]; col_bin
    [n_cols]."""
    scores = np.asarray(scores, np.float64)
    nm = scores.shape[1]
    n_cols = len(col_bin)
    best_v = [[[0.0] * nm for _ in range(B)] for _ in range(n_cols)]
    all_v = [[[(0.0, 0, 0)] * nm for _ in range(B)] for _ in range(n_cols)]
    for off, c0, F in segs:
        for b in range(B):
            for m in range(nm):
                v = [[float(scores[off + (j * B + b) * ns + s, m]) for j in range(F)] for s in range(ns)]
                s_best = best_ref(v, (higher_mask >> m) & 1)
                for j in range(F):
                    acc, n_inf, n_nan = 0.0, 0, 0
                    for s in range(ns):
                        a = v[s][j]
                        if math.isnan(a):
                            n_nan += 1
                        elif math.isinf(a):
                            n_inf += 1
                        else:
                            acc += a
                    best_v[c0 + j][b][m] = v[s_best][j]
                    all_v[c0 + j][b][m] = (acc, n_inf, n_nan)
    done = set()
    for c, u in enumerate(col_bin):
        if u in done:
            continue
        done.add(u)
        cols = [cc for cc in range(c, n_cols) if col_bin[cc] == u]
        tot["rows"][u] += B * len(cols)
        for m in range(nm):
            sb = sq = sa = 0.0
            cnt = [0, 0, 0, 0]
            for cc in cols:
                for b in range(B):
                    a = best_v[cc][b][m]
                    if math.isnan(a):
                        cnt[1] += 1
                    elif math.isinf(a):
                        cnt[0] += 1
                    else:
                        sb += a
                        sq += a * a
                    acc, n_inf, n_nan = all_v[cc][b][m]
                    sa += acc
                    cnt[2] += n_inf
                    cnt[3] += n_nan
            S = tot["sums"][u, m]
            S[0], S[1], S[2] = float(S[0]) + sb, float(S[1]) + sq, float(S[2]) + sa
            tot["counts"][u, m] += np.array(cnt, np.int64)
    return tot


def fold_results(tot, index, results, lens, nsample, names):
    """Adds the looped p2p_evaluate results of one batch (results[k]: the dict for length lens[k]) to tot in float64, with
    the best sample taken from each result's 'best' indices: the host aggregation evaluate_split stands for.  index maps
    (L, frame) -> bin and grows as plan_bins grows it; tot is grown to fit."""
    for L, r in zip(lens, results):
        for j, f in enumerate(r["frames"]):
            u = index.setdefault((int(L), int(f)), len(index))
            if u >= len(tot["rows"]):
                grow = new_totals(u + 1, len(names))
                for k in grow:
                    grow[k][:len(tot[k])] = tot[k]
                tot.update(grow)
            v = {k: r[k].double().cpu().numpy() for k in names}   # [nsample, F, B]
            B = v[names[0]].shape[2]
            tot["rows"][u] += B
            for m, k in enumerate(names):
                idx = r["best"][k][0].cpu().numpy()
                for b in range(B):
                    a = float(v[k][idx[b], j, b])
                    if math.isnan(a):
                        tot["counts"][u, m, 1] += 1
                    elif math.isinf(a):
                        tot["counts"][u, m, 0] += 1
                    else:
                        tot["sums"][u, m, 0] += a
                        tot["sums"][u, m, 1] += a * a
                    for s in range(nsample):
                        a = float(v[k][s, j, b])
                        if math.isnan(a):
                            tot["counts"][u, m, 3] += 1
                        elif math.isinf(a):
                            tot["counts"][u, m, 2] += 1
                        else:
                            tot["sums"][u, m, 2] += a
    return tot
