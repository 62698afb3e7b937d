"""Quantitative evaluation of a trained model over a test split: the numbers a video-generation paper reports, as one call.

``evaluate_split(model, batches, n_batches, len_outputs, nsample)`` scores n_batches test batches.  Per batch it runs ONE
``P2PModel.p2p_evaluate_lengths`` replay (every output length generated in one CUDA graph), ONE metrics launch over every
length's rows, and ONE p2pvg_metrics_fold launch (include/p2pvg_b200.h) that adds the batch to device-resident fp64 totals.
Nothing is read back until the end; then one device-to-host copy of the totals gives the report.

A bin is one (output length L, scored frame f) of the split.  A length equal to the batch's own length T scores every
generated frame n_past .. L - 1 against x[f]; any other length scores only its control point L - 1 against x[T - 1], in the
bin (L, L - 1).  With ``len_outputs=None`` each batch is generated at its own length, so dynamic-length test batches fill
the bins of every T that occurs.  Per bin and metric the fold keeps the sum over rows of the best sample's value (the sample
with the best mean over that length's scored frames, the first on ties: metrics.best_of's rule), its sum of squares, the
sum over rows and samples, and the +-inf and NaN values apart (PSNR is +inf for a frame identical to the ground truth); the
report gives means of the finite values and the share of infinite ones.

``python -m p2pvg_b200.evaluate --ckpt model.pth --data_root data [--nsample 20] [--lengths 10 20 30] [--n_batches N]
[--batch_size B] [--seed 1] [--out report.json]`` evaluates a checkpoint written by ``P2PModel.save`` on the test split of
its dataset (Moving MNIST, Weizmann or BAIR), built as the reference's data_utils builds it for train=False.
"""
from __future__ import annotations

import argparse
import json
import math
import random

import numpy as np
import torch

from . import metrics

# per bin and metric: fp64 sums (best, best^2, all samples) and int64 counts (best +-inf, best NaN, all +-inf, all NaN)
N_SUMS, N_COUNTS = 3, 4


def higher_mask(names):
    """p2pvg_metrics_fold's higher_mask: bit m set where a higher value of names[m] is better."""
    return sum(1 << m for m, k in enumerate(names) if metrics.HIGHER_IS_BETTER[k])


def plan_bins(lens, frames, offsets, index):
    """The fold tables of one batch scored by evaluate_lengths (lens in caller order, frames and offsets as
    score_lengths returns them): segs, per length (first pair, first column, scored frame count), and col_bin, per column
    (length k's frame j is column sum(len(frames[:k])) + j) the bin of (lens[k], frames[k][j]).  Bins not yet in index
    (a dict (L, f) -> bin) are appended to it in column order."""
    segs, col_bin = [], []
    for L, fk, off in zip(lens, frames, offsets):
        segs.append((off, len(col_bin), len(fk)))
        for f in fk:
            col_bin.append(index.setdefault((int(L), int(f)), len(index)))
    return segs, col_bin


class SplitTotals:
    """The device-resident totals of evaluate_split: one fp64 store holding sums [cap, nm, 3], counts (int64) [cap, nm, 4]
    and rows (int64) [cap], so that the report is one device-to-host copy.  Bins are numbered in order of first
    appearance; the store grows (on the device) when a batch brings new bins."""

    def __init__(self, names, device):
        from ._lib import kernels_for
        self.names, self.nm, self.dev = tuple(names), len(names), torch.device(device)
        self.K = kernels_for(self.dev)
        self.index, self.tables = {}, {}
        self.cap = 0
        self.store = torch.zeros(0, dtype=torch.float64, device=self.dev)
        self._views()
        self.counter = torch.zeros(1, dtype=torch.int32, device=self.dev)
        self.part_v = torch.zeros(0, dtype=torch.float64, device=self.dev)
        self.part_c = torch.zeros(0, dtype=torch.int32, device=self.dev)

    def _views(self):
        c, nm = self.cap, self.nm
        a, b = c * nm * N_SUMS, c * nm * (N_SUMS + N_COUNTS)
        self.sums = self.store[:a].view(c, nm, N_SUMS)
        self.counts = self.store[a:b].view(torch.int64).view(c, nm, N_COUNTS)
        self.rows = self.store[b:b + c].view(torch.int64)

    def _grow(self, n):
        if n <= self.cap:
            return
        old = (self.sums, self.counts, self.rows)
        self.cap = max(n, 2 * self.cap, 16)
        self.store = torch.zeros(self.cap * (self.nm * (N_SUMS + N_COUNTS) + 1), dtype=torch.float64, device=self.dev)
        self._views()
        for new, o in zip((self.sums, self.counts, self.rows), old):
            new[:len(o)].copy_(o)

    def fold(self, scores, lens, T, frames, offsets, B, nsample):
        """ONE p2pvg_metrics_fold launch of a batch's fp64 [n_pairs, nm] scores (frames, offsets: score_lengths' plan)."""
        key = (int(T), tuple(int(L) for L in lens), int(B), int(nsample))
        tabs = self.tables.get(key)
        if tabs is None:   # planned and checked once per (T, lengths, B, nsample)
            segs, col_bin = plan_bins(lens, frames, offsets, self.index)
            n_pairs = int(scores.shape[0])
            for off, c0, F in segs:
                if F < 1 or off < 0 or off + F * B * nsample > n_pairs or c0 + F > len(col_bin):
                    raise ValueError(f"fold plan does not fit the scores: segment ({off}, {c0}, {F}) of {n_pairs} pairs")
            tabs = self.tables[key] = (torch.tensor(segs, dtype=torch.int32).to(self.dev),
                                       torch.tensor(col_bin, dtype=torch.int32).to(self.dev))
        segs, col_bin = tabs
        self._grow(len(self.index))
        need = col_bin.numel() * B * self.nm * 2
        if self.part_v.numel() < need:
            self.part_v = torch.empty(need, dtype=torch.float64, device=self.dev)
            self.part_c = torch.empty(need, dtype=torch.int32, device=self.dev)
        self.K.metrics_fold(scores, higher_mask(self.names), B, nsample, segs, col_bin, self.part_v, self.part_c, self.counter,
                            self.sums, self.counts, self.rows)

    def read(self):
        """The totals on the host after ONE copy: (keys in bin order, sums [n, nm, 3], counts [n, nm, 4], rows [n])."""
        host = self.store.cpu().numpy()
        c, nm, n = self.cap, self.nm, len(self.index)
        a, b = c * nm * N_SUMS, c * nm * (N_SUMS + N_COUNTS)
        keys = sorted(self.index, key=self.index.get)
        return (keys, host[:a].reshape(c, nm, N_SUMS)[:n], host[a:b].view(np.int64).reshape(c, nm, N_COUNTS)[:n],
                host[b:b + c].view(np.int64)[:n])


def _num(v):
    """A finite float as is; None for a value that does not exist (JSON has no inf or NaN)."""
    return float(v) if v is not None and math.isfinite(v) else None


def bin_stats(s, n, rows, nsample):
    """One bin's report entry for one metric from its totals s = (best, best^2, all), n = (best inf, best NaN, all inf,
    all NaN) and row count."""
    nb = int(rows - n[0] - n[1])
    na = int(rows * nsample - n[2] - n[3])
    mean = s[0] / nb if nb else None
    sem = None
    if nb > 1:
        var = max((s[1] - s[0] * mean) / (nb - 1), 0.0)
        sem = math.sqrt(var / nb)
    return dict(best_mean=_num(mean), best_sem=_num(sem), mean=_num(s[2] / na if na else None),
                best_inf_share=float(n[0] / rows) if rows else None, inf_share=float(n[2] / (rows * nsample)) if rows else None,
                best_nan=int(n[1]), nan=int(n[3]))


def build_report(keys, sums, counts, rows, names, nsample, config):
    """The report of evaluate_split from the totals (SplitTotals.read): per bin (length, frame, rows and per metric
    bin_stats), per length (its frames, the best-sample mean pooled over its frames' finite values, the same over samples,
    and its control-point bin), and the PSNR inf shares pooled over every bin."""
    bins, lengths = [], {}
    for u in sorted(range(len(keys)), key=lambda u: keys[u]):
        L, f = keys[u]
        e = dict(length=L, frame=f, rows=int(rows[u]))
        for m, k in enumerate(names):
            e[k] = bin_stats(sums[u, m], counts[u, m], int(rows[u]), nsample)
        bins.append(e)
        lengths.setdefault(L, []).append(u)
    per_length = []
    for L, us in sorted(lengths.items()):
        e = dict(length=L, frames=[keys[u][1] for u in us])
        cp = next((u for u in us if keys[u][1] == L - 1), None)
        for m, k in enumerate(names):
            nb = sum(int(rows[u] - counts[u, m, 0] - counts[u, m, 1]) for u in us)
            na = sum(int(rows[u] * nsample - counts[u, m, 2] - counts[u, m, 3]) for u in us)
            sb = sum(float(sums[u, m, 0]) for u in us)
            sa = sum(float(sums[u, m, 2]) for u in us)
            e[k] = dict(best_mean_over_frames=_num(sb / nb if nb else None), mean_over_frames=_num(sa / na if na else None),
                        control_point=None if cp is None else _num(bin_stats(sums[cp, m], counts[cp, m], int(rows[cp]),
                                                                              nsample)["best_mean"]))
        per_length.append(e)
    report = dict(config=dict(config), metrics=list(names), bins=bins, lengths=per_length)
    if "psnr" in names:
        m = list(names).index("psnr")
        total = int(sum(int(r) for r in rows))
        report["psnr_inf_share"] = dict(best=float(counts[:, m, 0].sum() / total) if total else None,
                                        samples=float(counts[:, m, 2].sum() / (total * nsample)) if total else None)
    return report


def _backbone(model):
    if getattr(model, "is_pose", False):
        return "h36m_mlp"
    enc = model.encoder
    return f"{getattr(enc, 'backbone', 'dcgan')}_{enc.image_width}"


def evaluate_split(model, batches, n_batches, len_outputs=None, nsample=1, model_mode='full', data_range=1.0, seed=None):
    """Score n_batches batches of `batches` (any iterator of test batches: MovingMNIST, ClipBatches, PoseBatches, or a plain
    iterator of [T, B, ...] tensors or (pose_2d, pose_3d, camera_view) tuples) with best-of-nsample generation at every
    length of len_outputs (None: each batch's own length T).  Per batch one p2p_evaluate_lengths replay, one metrics launch
    and one p2pvg_metrics_fold launch; the host reads nothing until the end.  `seed`, the seed the caller drew the batches and
    noise from, is recorded in the report.  The same models as p2p_generate_graphed, in eval mode.

    Returns a JSON-ready dict (build_report): 'config' (nsample, lengths, batches, rows, seed, backbone, precision,
    model_mode, data_range), 'metrics', 'bins' (per (length, frame): rows and per metric the best-of-nsample mean and its
    standard error, the mean over samples, the inf shares and NaN counts), 'lengths' (per length its frames, the means
    over them and the control-point column) and, for frames, 'psnr_inf_share'.  Means are over finite values; None where
    there is none.  ValueError for n_batches < 1, nsample < 1 or batches that run out, and what p2p_evaluate_lengths
    rejects."""
    from . import infer
    if isinstance(n_batches, bool) or int(n_batches) != n_batches or n_batches < 1:
        raise ValueError(f"n_batches must be an int >= 1 (got {n_batches!r})")
    if isinstance(nsample, bool) or int(nsample) != nsample or nsample < 1:
        raise ValueError(f"nsample must be an int >= 1 (got {nsample!r})")
    eng = model._graphed_engine()
    it = iter(batches)
    totals, n_rows = None, 0
    for i in range(int(n_batches)):
        try:
            x = next(it)
        except StopIteration:
            raise ValueError(f"the batches ran out after {i} of {n_batches}") from None
        if isinstance(x, tuple):   # h36m: (pose_2d, pose_3d, camera_view) -> pose_3d
            x = x[1]
        T = len(x)
        lens = [T] if len_outputs is None else list(len_outputs)
        (frames, offsets, B), scores, names = eng.score_lengths(x, lens, int(nsample), model_mode, data_range)
        if totals is None:
            totals = SplitTotals(names, scores.device)
        totals.fold(scores, lens, T, frames, offsets, B, int(nsample))
        n_rows += B
    keys, sums, counts, rows = totals.read()
    config = dict(nsample=int(nsample), lengths=None if len_outputs is None else [int(L) for L in len_outputs],
                  batches=int(n_batches), rows=n_rows, seed=seed, backbone=_backbone(model),
                  precision="fp32" if infer._act_dtype() == torch.float32 else "bf16", model_mode=model_mode,
                  data_range=float(data_range))
    return build_report(keys, sums, counts, rows, totals.names, int(nsample), config)


# ------------------------------------------------------------------ command line
def parse_args(argv=None):
    p = argparse.ArgumentParser(description="Evaluate a P2PModel checkpoint on its dataset's test split: best-of-nsample "
                                            "SSIM, PSNR and MSE per output length and frame, written as a JSON report")
    p.add_argument('--ckpt', type=str, required=True, help='a model.pth written by P2PModel.save')
    p.add_argument('--data_root', type=str, default='', help="the dataset root (default: the checkpoint's opt.data_root)")
    p.add_argument('--nsample', type=int, default=20, help='samples per test sequence; the best one is scored')
    p.add_argument('--lengths', type=int, nargs='+', default=None,
                   help="output lengths to generate (default: each batch's own length)")
    p.add_argument('--n_batches', type=int, default=None, help='test batches to score (default: one pass over the split)')
    p.add_argument('--batch_size', type=int, default=None, help="default: the checkpoint's opt.batch_size")
    p.add_argument('--seed', type=int, default=1, help='seed of random, NumPy, torch and CUDA')
    p.add_argument('--out', type=str, default='report.json')
    args = p.parse_args(argv)
    if args.nsample < 1:
        p.error(f"--nsample must be >= 1 (got {args.nsample})")
    if args.n_batches is not None and args.n_batches < 1:
        p.error(f"--n_batches must be >= 1 (got {args.n_batches})")
    if args.batch_size is not None and args.batch_size < 1:
        p.error(f"--batch_size must be >= 1 (got {args.batch_size})")
    if args.lengths is not None and any(L < 2 for L in args.lengths):
        p.error(f"every --lengths entry must be >= 2 (got {args.lengths})")
    return args


def check_dataset(opt):
    """ValueError for a checkpoint whose test split the command line cannot build (h36m)."""
    if opt.dataset == "h36m":
        raise ValueError("h36m checkpoints are evaluated from Python: build PoseBatches from the reference's Human36mDataset "
                         "test split and call p2pvg_b200.evaluate.evaluate_split(model, batches, n_batches, ...) (see "
                         "INTEGRATION.md)")
    if opt.dataset not in ("mnist", "weizmann", "bair"):
        raise ValueError(f"unknown dataset {opt.dataset!r}")


def split_batches(opt, data_root, batch_size):
    """The test split's batches as the reference's data_utils builds them for train=False, and the batch count of one pass
    over it: (iterator, n_batches)."""
    from .data import ClipBatches, MovingMNIST, load_bair_clips, load_mnist_digits, load_weizmann_clips
    check_dataset(opt)
    if opt.dataset == "mnist":
        digits = load_mnist_digits(data_root, train=False)
        return (MovingMNIST(digits, batch_size, opt.max_seq_len, opt.delta_len, image_size=opt.image_width,
                            num_digits=opt.num_digits), max(len(digits) // batch_size, 1))
    if opt.dataset == "weizmann":   # data_utils.py: test_max_seq_len 10, lengths 6 .. 10
        clips = load_weizmann_clips(data_root, False, 10, opt.image_width)
        b = ClipBatches(clips, batch_size, "permutation", (6, 10))
    else:
        clips = load_bair_clips(data_root, False, opt.max_seq_len, opt.image_width)
        b = ClipBatches(clips, batch_size, "ordered", (opt.max_seq_len - 2 * opt.delta_len, opt.max_seq_len))
    return b, b.epoch_batches


def main(argv=None):
    args = parse_args(argv)
    from .generate import backbone_of
    from .models.p2p_model import P2PModel
    states = torch.load(args.ckpt, weights_only=False)
    opt = states['opt']
    try:
        check_dataset(opt)
    except ValueError as e:
        raise SystemExit(f"p2pvg_b200.evaluate: {e}") from None
    opt.backbone_net = backbone_of(opt)
    random.seed(args.seed)
    np.random.seed(args.seed)
    torch.manual_seed(args.seed)
    torch.cuda.manual_seed_all(args.seed)
    B = args.batch_size or int(opt.batch_size)
    model = P2PModel(B, opt.channels, opt.g_dim, opt.z_dim, opt.rnn_size, opt.prior_rnn_layers, opt.posterior_rnn_layers,
                     opt.predictor_rnn_layers, opt=opt)
    model.cuda()
    model.load(states=states)
    model.eval()
    batches, n = split_batches(opt, args.data_root or opt.data_root, B)
    report = evaluate_split(model, batches, args.n_batches or n, args.lengths, args.nsample, seed=args.seed)
    with open(args.out, "w") as f:
        json.dump(report, f, indent=1)
        f.write("\n")
    return report


if __name__ == "__main__":
    main()
