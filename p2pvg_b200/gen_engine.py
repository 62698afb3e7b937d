"""Graph-captured point-to-point generation for the dcgan, vgg and h36m_mlp backbones (reference models/p2p_model.py:80-183).

The recurrent part and all host logic below are shared; the backbone-specific parts (model check, weight preparation,
encode, skip halves, decode, the frame shape) are methods that ``PoseGenerateEngine`` (at the end of this file) and
``gen_engine_vgg.VggGenerateEngine`` (vgg_64 / vgg_128) override.  For poses every encoder and decoder call is one
p2pvg_pose_mlp launch, so an executed autoregressive step is at most four launches.

``GenerateEngine`` computes what ``infer.p2p_generate`` / ``infer.p2p_generate_samples`` compute, with every call one
replay of a CUDA graph captured per signature (rows, sequence lengths, executed steps, model_mode, n_past,
last_frame_skip, precision and the device addresses of every parameter and BatchNorm buffer read).

Host work per call: the reference's NumPy skip draw, the slot planner below, the per-slot tables (time_until_cp,
delta_time, posterior target), the eps buffer, the replay, and copying the generated frames out of graph memory.
Inside the graph:
  * the bf16 weight packs and the eval-BatchNorm coefficients are recomputed from the live parameters, so a training
    step between two calls is picked up without any host bookkeeping;
  * the ground-truth frames are encoded once, time-batched at B rows (not nsample * B; eval-mode rows are independent);
    that one encode gives global_z, the posterior targets, the teacher-forced inputs and the skip maps;
  * the skip half of every decoder torch.cat([d, skip]) is computed once per call (per decode when last_frame_skip);
  * every executed slot runs the encoder on the previous decoded frame (only after the teacher-forced steps), the
    posterior, prior and frame predictor, and the decoder.

Recurrent part: per executed step ONE p2pvg_lstm_step launch for posterior + prior and one for the frame predictor (embed,
LSTM cells with the state updated in place, heads and reparameterisation in one kernel; exact fp32 in both precisions, as
the eager path's LSTMs).  The module inputs torch.cat([h, global_z | z, tuc, dt]) are read through per-slot index tables.

Layer dispatch (bf16 mode): the 4x4/s2 convolutions with >= 64 channels on both sides are implicit GEMMs
(p2pvg_conv_gemm kinds 0 / 2) with eval-BatchNorm + activation in their epilogue; the thin 1- / 3-channel ends
(im2col / col2im + GEMM), the 4x4-valid GEMMs (encoder final, decoder first) and all of the fp32 mode use the explicit
lowering followed by p2pvg_bn_act, as infer.py does (the training engine lowers the thin ends the same way).

``generate_multi_cp`` (P2PModel.p2p_generate_multi_cp) replays a chain of segments x[cp_ixs[k] : cp_ixs[k + 1] + 1], each
what one call with init_hidden=False after the first computes; a single call is the one-segment chain.  The per-slot tables
(plan_segments) index clip frames, so every slot reads its segment's ground truth, global descriptor (a per-slot tab_int
entry) and counters; the LSTM state stays in the graph's buffers across segments.  A chain's ground-truth encode covers the
clip followed by a copy of each segment's skip source frame, so that the skip halves of all segments are one batched launch
per stage, of which each decode reads its segment's B images.

``generate_lengths`` (P2PModel.p2p_generate_lengths) replays one call per output length as ONE graph: each length owns a
group of nsample * B rows, the groups sorted longest first (plan_lengths), so that the rows still generating at step i are a
prefix of the batch and every launch of step i runs on that prefix only.  A length changes only the time counters (one
tab_f entry per slot and group, read per row through p2pvg_lstm_step's counter_rows) and the step where its rows stop; the
other tables are the longest length's.  The module inputs are indexed with the step's row count as stride, so the ground
truth h source is kept once per distinct active row count; every other buffer is allocated at its first, largest use.

``evaluate`` (P2PModel.p2p_evaluate) runs the replay of a generate call (or chain) and, instead of assembling the output list,
scores the decoded frames in the graph's output buffer against the ground truth in its input buffer with one metrics launch
(metrics.plan_pairs / plan_pairs_multi_cp name the rows).  ``evaluate_lengths`` (P2PModel.p2p_evaluate_lengths) does the
same for every length of one generate_lengths replay: one metrics launch over all row groups (metrics.plan_pairs_lengths).

Memory: every cached signature (at most MAX_GRAPHS, least recently used evicted) owns its buffers; the ground-truth encode
covers all len(x) frames of the call.  ``GenerateEngine.memory_bytes()`` reports the total, ``clear()`` frees it.

Noise: eps comes from ONE torch.randn of shape [slots, 2, rows, z] per call, so for a given torch seed the values
differ from the eager path's per-step draws (the distribution is the same).  Inside ``infer.eps_stream`` the injected
draws are consumed in the reference's order (posterior, then prior, per executed step).
"""
from __future__ import annotations

from collections import OrderedDict

import numpy as np
import torch

from ._lib import ACT_LRELU, ACT_SIGMOID, ACT_TANH
from .engine import capture_graph
from .layouts import cast, implicit_shape, nchw_to_nhwc, nhwc_to_nchw, pack_conv4, pack_convt4, tile_bias

MAX_GRAPHS = 4


def plan_slots(len_output, len_x, probs, skip_prob, n_past, skip_frame, eval_cp_ix):
    """Executed steps of p2p_generate (reference models/p2p_model.py:126-138): a list of (i, time_until_cp, delta_time,
    target) per executed step i, in Python doubles exactly as the reference computes them; target = i while a
    ground-truth frame x[i] exists, else -1 (the posterior then reads h_cpaw, :167-171)."""
    prev_i, skip_count, out = 0, 0, []
    max_skip_count = len_x * skip_prob
    for i in range(1, len_output):
        if (probs[i - 1] <= skip_prob and i >= n_past and skip_count < max_skip_count and i != 1
                and i != (len_output - 1) and skip_frame):
            skip_count += 1
            continue
        out.append((i, (eval_cp_ix - i + 1) / eval_cp_ix, (i - prev_i) / eval_cp_ix, i if i < len_x else -1))
        prev_i = i
    return out


def plan_segments(segs, T, probs, skip_prob, n_past, skip_frame, model_mode):
    """Executed steps and per-slot tables of a chain of generate calls whose inputs are slices of one clip.

    segs: per segment (offset, T_k, L_k, eval_cp_ix_k): the call p2p_generate(x[offset : offset + T_k], L_k, eval_cp_ix_k);
    probs: each segment's NumPy skip draw; T: the clip's frame count, which is also the index of the row that holds the
    autoregressive encode in the engine's h source.  The slots of all segments are numbered in chain order.

    Returns (slots, ints, floats): plan_slots of each segment; the int32 table [tab_i | tab_h | tab_z | tab_g] of 4 * S
    entries (clip frame of the posterior target, clip frame or T of the encoder input h, 0 / 1 for the predictor's z from
    the posterior / prior, clip frame of the global descriptor); the float table [time_until_cp | delta_time] of 2 * S."""
    slots, tab_i, tab_h, tab_z, tab_g, tuc, dt = [], [], [], [], [], [], []
    for (o, Tk, Lk, cp), pr in zip(segs, probs):
        sl = plan_slots(Lk, Tk, pr, skip_prob, n_past, skip_frame, cp)
        n_tf = min(n_past - 1, Lk - 1)
        slots.append(sl)
        for j, (_, t, d, tgt) in enumerate(sl):
            h = o + j if j <= n_tf else T                  # ground truth until the segment's first decode
            tab_h.append(h)
            tab_i.append(o + tgt if tgt >= 0 else h)       # posterior: x_k[i], or h_cpaw's h when x_k has no frame i
            tab_z.append(0 if (model_mode == "posterior" or (j < n_tf and model_mode == "full")) else 1)
            tab_g.append(o + Tk - 1)                       # global descriptor: the segment's control point
            tuc.append(t)
            dt.append(d)
    return slots, tab_i + tab_h + tab_z + tab_g, tuc + dt


def check_cp_ixs(cp_ixs, T, len_outputs, n_past):
    """The segments (offset, T_k, L_k, L_k - 1) of a multi-control-point call on a clip of T frames; ValueError for a
    malformed cp_ixs or len_outputs, or a segment with fewer than min(n_past, L_k) frames."""
    try:
        cps = [int(v) for v in cp_ixs]
    except (TypeError, ValueError):
        raise ValueError(f"cp_ixs must be a sequence of ints (got {cp_ixs!r})") from None
    if any(isinstance(v, bool) or int(v) != v for v in cp_ixs):
        raise ValueError(f"cp_ixs must be a sequence of ints (got {cp_ixs!r})")
    if len(cps) < 2 or cps[0] != 0 or any(b <= a for a, b in zip(cps, cps[1:])) or cps[-1] > T - 1:
        raise ValueError(f"cp_ixs must start at 0, increase strictly, have at least 2 entries and end at or before the last "
                         f"input frame {T - 1} (got {cps})")
    Ts = [b - a + 1 for a, b in zip(cps, cps[1:])]
    if len_outputs is None:
        Ls = Ts
    else:
        Ls = list(len_outputs)
        if len(Ls) != len(Ts):
            raise ValueError(f"len_outputs needs one entry per segment ({len(Ts)}), got {len(Ls)}")
        if any(isinstance(v, bool) or int(v) != v or v < 2 for v in Ls):
            raise ValueError(f"every len_outputs entry must be an int >= 2 (got {Ls})")
        Ls = [int(v) for v in Ls]
    for k, (Tk, Lk) in enumerate(zip(Ts, Ls)):
        if n_past < 1 or Tk < min(n_past, Lk):
            raise ValueError(f"segment {k} has {Tk} frames; it needs n_past >= 1 and at least min(n_past, len_output) = "
                             f"{min(n_past, Lk)}")
    return [(o, Tk, Lk, Lk - 1) for o, Tk, Lk in zip(cps, Ts, Ls)]


def check_lengths(len_outputs, T, n_past):
    """The output lengths of a generate_lengths call on a clip of T frames as a list of ints; ValueError for an empty or
    malformed len_outputs, a length below 2, or a length L with T < min(n_past, L)."""
    try:
        Ls = list(len_outputs)
        bad = not Ls or any(isinstance(v, bool) or int(v) != v or v < 2 for v in Ls)
    except (TypeError, ValueError):
        bad = True
    if bad:
        raise ValueError(f"len_outputs must be a non-empty sequence of ints >= 2 (got {len_outputs!r})")
    Ls = [int(v) for v in Ls]
    for L in Ls:
        if n_past < 1 or T < min(n_past, L):
            raise ValueError(f"len_output {L} needs n_past >= 1 and at least min(n_past, len_output) = {min(n_past, L)} input "
                             f"frames (got {T})")
    return Ls


def lengths_order(lens):
    """The row groups of generate_lengths: caller indices sorted by length, longest first, ties in caller order."""
    return sorted(range(len(lens)), key=lambda k: -lens[k])


def plan_lengths(lens, len_x, probs, skip_prob, n_past, group_rows):
    """The ragged rows of generate_lengths: output length lens[k] is row group order.index(k) (lengths_order) of group_rows
    rows.  Step i (slot i - 1) runs on the groups whose length is greater than i, which are a prefix of the rows.

    Returns (order, active, floats): the caller index of every group; the active row count of every slot; the float table
    [time_until_cp | delta_time] of 2 * S * G entries, slot-major, with group g's counters at slot s * G + g (plan_slots'
    doubles for its own length; zero once the group has stopped)."""
    order = lengths_order(lens)
    nG, S = len(lens), max(lens) - 1
    active = [group_rows * sum(1 for L in lens if L > i) for i in range(1, S + 1)]
    tuc, dt = [0.0] * (S * nG), [0.0] * (S * nG)
    for g, k in enumerate(order):
        for s, (_, t, d, _) in enumerate(plan_slots(lens[k], len_x, probs[k], skip_prob, n_past, False, lens[k] - 1)):
            tuc[s * nG + g], dt[s * nG + g] = t, d
    return order, active, tuc + dt


def check_supported(model):
    """ValueError unless the model is a dcgan_64 / dcgan_128 P2PModel with every module in eval mode."""
    from .models.backbone import DcganDecoder, DcganEncoder
    if getattr(model, "is_pose", False) or not isinstance(model.encoder, DcganEncoder) or not isinstance(model.decoder, DcganDecoder):
        raise ValueError("p2p_generate_graphed supports the dcgan_64 / dcgan_128, vgg_64 / vgg_128 and h36m_mlp backbones only; use "
                         "p2p_generate for this model")
    _check_eval(model)


def check_supported_pose(model):
    """ValueError unless the model is an h36m_mlp P2PModel in eval mode whose LSTMs p2pvg_lstm_step runs."""
    from .models.h36m_mlp import decoder, encoder
    if not getattr(model, "is_pose", False) or not isinstance(model.encoder, encoder) or not isinstance(model.decoder, decoder):
        raise ValueError("PoseGenerateEngine runs the h36m_mlp backbone only; use p2p_generate for this model")
    _check_eval(model)
    R = int(model.rnn_size)
    if not (64 <= R <= 512 and R % 8 == 0):
        raise ValueError(f"p2p_generate_graphed runs rnn_size 64..512 in multiples of 8 (got {R}); use p2p_generate")


def _check_eval(model):
    for m in ("encoder", "decoder", "frame_predictor", "posterior", "prior"):
        if any(mod.training for mod in getattr(model, m).modules()):
            raise ValueError(f"p2p_generate_graphed needs every module in eval mode ({m} is in training mode); "
                             "call model.eval() or use p2p_generate")


class _Graph:
    def __init__(self):
        self.bufs = {}
        self.graph = None
        self.ws_gen = None
        self.eval_lengths = {}   # evaluate_lengths' pair plans, per len_outputs in caller order


class GenerateEngine:
    def __init__(self, model):
        self.model = model
        self._graphs = OrderedDict()

    # ------------------------------------------------------------------ public entry
    @torch.no_grad()
    def generate(self, x, len_output, eval_cp_ix, model_mode="full", skip_frame=False, init_hidden=True, nsample=1):
        if isinstance(x, tuple):   # h36m: (pose_2d, pose_3d, camera_view) -> pose_3d (models/p2p_model.py:96-103)
            x = x[1]
        G, slots = self._replay(x, len_output, eval_cp_ix, model_mode, skip_frame, init_hidden, nsample)
        return self._assemble(G, x, slots[0], len_output)

    @torch.no_grad()
    def generate_multi_cp(self, x, cp_ixs, len_outputs=None, model_mode="full", skip_frame=False, nsample=1):
        """The chain generate(x_0, L_0, L_0 - 1, init_hidden=True), then generate(x_k, L_k, L_k - 1, init_hidden=False) for
        k >= 1, with x_k = x[cp_ixs[k] : cp_ixs[k + 1] + 1], as ONE replay: see P2PModel.p2p_generate_multi_cp."""
        if isinstance(x, tuple):
            x = x[1]
        G, slots, segs = self._replay_chain(x, cp_ixs, len_outputs, model_mode, skip_frame, nsample)
        out, res, d = G.bufs["out"].clone(), [], 0
        for (o, Tk, Lk, _), sl, (_, _, _, Sk, n_tf) in zip(segs, slots, G.cfg["segs"]):
            n_dec = max(Sk - n_tf, 0)
            res.append(self._assemble_seq(G.cfg, out[d:d + n_dec], x[o:o + Tk], sl, Lk))
            d += n_dec
        return res

    @torch.no_grad()
    def generate_lengths(self, x, len_outputs, model_mode="full", nsample=1):
        """generate(x, L, L - 1, model_mode, skip_frame=False, nsample=nsample) for every L in len_outputs, in order, as ONE
        replay: see P2PModel.p2p_generate_lengths."""
        if isinstance(x, tuple):
            x = x[1]
        G, slots, lens, order = self._replay_lengths(x, len_outputs, model_mode, nsample)
        c = G.cfg
        out, gr = G.bufs["out"].clone(), c["grows"]
        res = []
        for k, L in enumerate(lens):
            g = order.index(k)
            res.append(self._assemble_seq(dict(c, rows=gr), out[:, g * gr:(g + 1) * gr], x, slots[0][:L - 1], L))
        return res

    @torch.no_grad()
    def evaluate(self, x, nsample=1, len_output=None, model_mode="full", data_range=1.0, cp_ixs=None):
        """generate(x, L, L - 1, model_mode, skip_frame=False, nsample=nsample) with L = len_output or len(x) (or, given cp_ixs,
        generate_multi_cp(x, cp_ixs, None, model_mode, skip_frame=False, nsample=nsample)), scored by ONE metrics launch on the
        graph's own output and input buffers (metrics.plan_pairs / plan_pairs_multi_cp): see P2PModel.p2p_evaluate."""
        from . import metrics
        if isinstance(x, tuple):
            x = x[1]
        self._check_model()
        T = len(x)
        n_past = int(self.model.opt.n_past)
        if cp_ixs is not None:
            if len_output is not None:
                raise ValueError("p2p_evaluate takes cp_ixs or len_output, not both (with cp_ixs every segment keeps the clip's "
                                 "timing)")
            segs = check_cp_ixs(cp_ixs, T, None, n_past)
            for k, (_, _, Lk, _) in enumerate(segs):
                if Lk <= n_past:
                    raise ValueError(f"p2p_evaluate: segment {k} generates nothing to score ({Lk} frames <= n_past = {n_past})")
            metrics._check_range(data_range)
            G, _, _ = self._replay_chain(x, cp_ixs, None, model_mode, False, nsample)
        else:
            L = T if len_output is None else int(len_output)
            if L <= n_past:
                raise ValueError(f"p2p_evaluate: nothing is generated to score (len_output = {L} <= n_past = {n_past})")
            metrics._check_range(data_range)
            G, _ = self._replay(x, L, L - 1, model_mode, False, True, nsample)
        c = G.cfg
        B, fshape = c["B"], c["fshape"]
        pairs = G.bufs.get("eval_pairs")
        if pairs is None:   # the plan depends on nothing but the graph's signature
            if cp_ixs is not None:
                frames, pairs = metrics.plan_pairs_multi_cp([o for (o, _, _, _, _) in c["segs"]] + [c["T"] - 1], n_past, nsample, B)
            else:
                frames, pairs = metrics.plan_pairs(L, T, n_past, nsample, B)
            pairs = G.bufs["eval_pairs"] = pairs.to(c["dev"])
            G.eval_frames = frames
        frames = G.eval_frames
        out, xb = G.bufs["out"], G.bufs["x"]
        if self.model.is_pose:
            res, names = metrics.launch_pose_metrics(out, xb, pairs, fshape[0]), metrics.POSE_METRICS
        else:
            res, names = metrics.launch_frame_metrics(out, xb, pairs, fshape, data_range), metrics.FRAME_METRICS
        res = res.view(len(frames), B, nsample, len(names)).permute(3, 2, 0, 1)   # [metric][sample][frame][b]
        scores = {k: res[i].contiguous() for i, k in enumerate(names)}
        return dict(frames=list(frames), **scores, best=metrics.best_of(scores, names))

    @torch.no_grad()
    def evaluate_lengths(self, x, len_outputs, nsample=1, model_mode="full", data_range=1.0):
        """evaluate(x, nsample, L, model_mode, data_range) for every L in len_outputs, in order, from ONE generate_lengths
        replay and ONE metrics launch (score_lengths): see P2PModel.p2p_evaluate_lengths."""
        from . import metrics
        (frames, offsets, B), res, names = self.score_lengths(x, len_outputs, nsample, model_mode, data_range)
        out = []
        for fk, o in zip(frames, offsets):
            r = res[o:o + len(fk) * B * nsample].view(len(fk), B, nsample, len(names)).permute(3, 2, 0, 1)
            scores = {k: r[i].contiguous() for i, k in enumerate(names)}
            out.append(dict(frames=list(fk), **scores, best=metrics.best_of(scores, names)))
        return out

    @torch.no_grad()
    def score_lengths(self, x, len_outputs, nsample=1, model_mode="full", data_range=1.0):
        """The replay of generate_lengths(x, len_outputs, model_mode, nsample), then ONE metrics launch that scores every
        length's row group in the graph's own output and input buffers (metrics.plan_pairs_lengths, planned once per graph
        signature and len_outputs).  ValueError before any draw or launch for what check_lengths rejects, a length <= n_past
        or a data_range that is not positive.  Returns ((frames, offsets, B), scores, names): per length its scored frames and
        first pair and the batch size, the fp64 [n_pairs, len(names)] scores on the device, and the metric names."""
        from . import metrics
        if isinstance(x, tuple):
            x = x[1]
        self._check_model()
        T, n_past = len(x), int(self.model.opt.n_past)
        lens = check_lengths(len_outputs, T, n_past)
        for L in lens:
            if L <= n_past:
                raise ValueError(f"p2p_evaluate_lengths: nothing is generated to score (len_output = {L} <= n_past = {n_past})")
        metrics._check_range(data_range)
        G, _, _, _ = self._replay_lengths(x, lens, model_mode, nsample)
        c = G.cfg
        plan = G.eval_lengths.get(tuple(lens))
        if plan is None:   # the plan depends on nothing but the graph's signature and the caller's order of the lengths
            frames, pairs, offsets = metrics.plan_pairs_lengths(lens, T, n_past, nsample, c["B"])
            plan = G.eval_lengths[tuple(lens)] = (frames, pairs.to(c["dev"]), offsets)
        frames, pairs, offsets = plan
        out, xb = G.bufs["out"], G.bufs["x"]
        if self.model.is_pose:
            res, names = metrics.launch_pose_metrics(out, xb, pairs, c["fshape"][0]), metrics.POSE_METRICS
        else:
            res, names = metrics.launch_frame_metrics(out, xb, pairs, c["fshape"], data_range), metrics.FRAME_METRICS
        return (frames, offsets, c["B"]), res, names

    @torch.no_grad()
    def vis_canvas(self, x, len_output, model_mode, nsample, plan):
        """vis_seq's generation and composition (p2pvg_b200.visualize): the replay of generate(x, len_output, len_output - 1,
        model_mode, skip_frame=False, nsample=nsample), then ONE p2pvg_vis_canvas launch that reads the graph's own input and
        output buffers (no copy of the generated frames).  plan(gt_ref, sample_ref) returns the tile table (see
        visualize.plan_tiles); gt_ref(t) and sample_ref(s, t) give (store, frame of row 0) of ground-truth frame t and of
        sample s's frame t, sample_ref None for a skipped (zero) frame.  Returns visualize.compose's (canvas, video, gif)."""
        from . import visualize
        G, slots = self._replay(x, len_output, len_output - 1, model_mode, False, True, nsample)
        c = G.cfg
        B, rows, n_past = c["B"], c["rows"], c["n_past"]
        dec, d = {}, 0
        for (i, _, _, _) in slots[0]:
            if i >= n_past:
                dec[i] = d
                d += 1
        executed = {i for (i, _, _, _) in slots[0]}

        def sample_ref(s, t):
            if t == 0 or (t in executed and t < n_past):
                return 0, t * B
            if t not in executed:
                return None
            return 1, dec[t] * rows + s * B

        tiles = plan(lambda t: (0, t * B), sample_ref)
        return visualize.compose(G.bufs["x"], G.bufs["out"], tiles, c["fshape"][0], c["W"])

    def _replay(self, x, len_output, eval_cp_ix, model_mode, skip_frame, init_hidden, nsample):
        """One call: the one-segment chain over all len(x) frames.  Returns the graph and [executed slots]."""
        return self._run(x, len(x), [(0, len(x), len_output, eval_cp_ix)], model_mode, skip_frame, init_hidden, nsample)

    def _replay_lengths(self, x, len_outputs, model_mode, nsample):
        """A generate_lengths call: checks before any draw or launch, then the one-segment plan of the longest length over
        row groups of every length.  Returns the graph, [executed slots of the longest length], the lengths and the group
        order (lengths_order)."""
        self._check_model()
        lens = check_lengths(len_outputs, len(x), int(self.model.opt.n_past))
        Lmax = max(lens)
        G, slots = self._run(x, len(x), [(0, len(x), Lmax, Lmax - 1)], model_mode, False, True, nsample, lens=lens)
        return G, slots, lens, lengths_order(lens)

    def _replay_chain(self, x, cp_ixs, len_outputs, model_mode, skip_frame, nsample):
        """A multi-control-point call: checks before any draw or launch, then the chain of segments (offset, T_k, L_k,
        L_k - 1) over the clip's first cp_ixs[-1] + 1 frames.  Returns the graph, the slots per segment and the segments."""
        self._check_model()
        segs = check_cp_ixs(cp_ixs, len(x), len_outputs, int(self.model.opt.n_past))
        T = segs[-1][0] + segs[-1][1]
        G, slots = self._run(x, T, segs, model_mode, skip_frame, True, nsample)
        return G, slots, segs

    def _run(self, x, T, segs, model_mode, skip_frame, init_hidden, nsample, lens=None):
        """Steps (1)-(5) of a chain of segments (offset, T_k, L_k, eval_cp_ix_k) on the clip x[:T]: capture on first use of
        the signature, write this call's inputs, replay, and leave the LSTM state in the modules' .hidden as the eager path
        does.  Returns the graph and the executed slots of each segment.

        lens (generate_lengths; one segment of the longest length, skip_frame False): one row group of nsample * B rows per
        output length (plan_lengths), each with its own NumPy draw, counters and eps; .hidden is left holding the group of
        lens[-1]."""
        from . import infer
        model = self.model
        self._check_model()
        if model_mode not in ("full", "posterior", "prior"):
            raise ValueError(f"unknown model_mode {model_mode!r}")
        if nsample < 1:
            raise ValueError("nsample must be >= 1")
        opt = model.opt
        fshape = self._frame_shape(x[0])
        B = int(x[0].shape[0])
        n_past = int(opt.n_past)
        if n_past < 1 or any(Tk < min(n_past, Lk) for (_, Tk, Lk, _) in segs):
            raise ValueError("p2p_generate_graphed needs n_past >= 1 and at least min(n_past, len_output) input frames")
        nG = 1 if lens is None else len(lens)
        grows = nsample * B   # rows of one output length
        rows = nG * grows
        dev = x[0].device
        # (1) the reference's NumPy draw per segment (per output length), made even when skip_frame is False
        # (models/p2p_model.py:128)
        if lens is None:
            probs = [np.random.uniform(0, 1, Lk - 1) for (_, _, Lk, _) in segs]
            slots, ints, fl = plan_segments(segs, T, probs, float(opt.skip_prob), n_past, skip_frame, model_mode)
            order, feed = [0], None
        else:
            probs = [np.random.uniform(0, 1, L - 1) for L in lens]
            order, active, fl = plan_lengths(lens, T, probs, float(opt.skip_prob), n_past, grows)
            # the tables the groups share (targets, encoder inputs, z source, global descriptor): the longest length's
            slots, ints, _ = plan_segments(segs, T, [probs[order[0]]], float(opt.skip_prob), n_past, False, model_mode)
            feed = [(order.index(k), L - 1) for k, L in enumerate(lens)]   # (group, executed steps) in caller order
        Ss = [len(sl) for sl in slots]
        S = sum(Ss)
        if lens is None or nG == 1:
            active = [rows] * S
        feed = feed or [(0, S)]
        lfs = bool(opt.last_frame_skip)
        adt = infer._act_dtype()
        K = infer.kernels_for(dev)
        ptrs = tuple(p.data_ptr() for p in model.parameters()) + tuple(b.data_ptr() for b in model.buffers())
        # one segment: (len_output, executed steps), as for a single call; a chain: (T_k, L_k, S_k) per segment
        seg_sig = (segs[0][2], S) if len(segs) == 1 else (tuple((Tk, Lk, Sk) for (_, Tk, Lk, _), Sk in zip(segs, Ss)),)
        if nG > 1:   # generate_lengths: the graph depends on the lengths in group order
            seg_sig += (tuple(lens[k] for k in order),)
        sig = (rows, B, T, fshape, *seg_sig, model_mode, n_past, lfs, str(adt), ptrs)
        G = self._graphs.get(sig)
        if G is not None and G.ws_gen != K.ws_gen:
            del self._graphs[sig]
            G = None
        cseg = tuple((o, Tk, Lk, Sk, min(n_past - 1, Lk - 1)) for (o, Tk, Lk, _), Sk in zip(segs, Ss))
        # the ground-truth frames whose skip maps give the decoders' skip halves, one per segment: x_k[max(n_past - 2, 0)],
        # or with last_frame_skip the frame before the segment's first decode.  One segment reads it in place; a chain
        # appends copies of them behind the clip, so that all segments' skip halves come from one batched launch per stage
        src = [o + min(n_tf if lfs else max(n_past - 2, 0), Tk - 1) for (o, Tk, _, _, n_tf) in cseg]
        cfg = dict(rows=rows, grows=grows, nG=nG, active=tuple(active), B=B, T=T, fshape=fshape, C=fshape[0], W=fshape[-1], S=S, segs=cseg, src=src,
                   T_enc=T if len(segs) == 1 else T + len(segs), n_dec=sum(max(Sk - n_tf, 0) for (_, _, _, Sk, n_tf) in cseg),
                   mode=model_mode, n_past=n_past, lfs=lfs, adt=adt, ns=nsample, dev=dev)
        if not init_hidden:
            for m in ("posterior", "prior", "frame_predictor"):
                mod = getattr(model, m)
                if mod.hidden is None or len(mod.hidden) != mod.n_layers or tuple(mod.hidden[0][0].shape) != (rows, mod.hidden_size):
                    raise ValueError(f"init_hidden=False needs {m}.hidden of shape [{rows}, {mod.hidden_size}] per layer")
        # capture on first use of a signature, after one eager warm-up run of the same sequence.  This comes BEFORE the inputs
        # of the call are written: the graph updates the LSTM state buffers in place, so the warm-up and capture must not
        # run on the state this call starts from
        if G is None:
            G = _Graph()
            G.cfg = cfg
            self._alloc_io(G)
            self._body(G)
            G.graph = capture_graph(lambda: self._body(G), dev)
            G.ws_gen = K.ws_gen
            self._graphs[sig] = G
            while len(self._graphs) > MAX_GRAPHS:
                self._graphs.popitem(last=False)
        else:
            self._graphs.move_to_end(sig)
        # (2)-(4) inputs of this call: frames, per-slot tables, eps, initial LSTM state
        xs = x if torch.is_tensor(x) else torch.stack(list(x))
        xb = G.bufs["x"].view(cfg["T_enc"], B, *fshape)
        xb[:T].copy_(xs[:T].reshape(T, B, *fshape))
        if cfg["T_enc"] > T:
            xb[T:].copy_(xs[src].reshape(len(src), B, *fshape))
        G.bufs["tab_int"][:4 * S].copy_(torch.tensor(ints, dtype=torch.int32), non_blocking=True)
        G.bufs["tab_f"][:2 * S * nG].copy_(torch.tensor(fl, dtype=torch.float64).float(), non_blocking=True)
        if S:
            z = model.z_dim
            if infer._EPS_STREAM is not None:
                for g, Sg in feed:
                    for s in range(Sg):
                        for j in (0, 1):
                            G.bufs["eps"][s, j, g * grows:(g + 1) * grows].copy_(
                                infer._EPS_STREAM.pop(0).to(device=dev, dtype=torch.float32).reshape(grows, z))
            else:
                torch.randn(S, 2, rows, z, device=dev, out=G.bufs["eps"])
        for m in ("posterior", "prior", "frame_predictor"):
            hs, cs = G.bufs[f"{m}_h"], G.bufs[f"{m}_c"]
            if init_hidden:
                hs.zero_()
                cs.zero_()
            else:
                for l, (h, c) in enumerate(getattr(model, m).hidden):
                    hs[l].copy_(h)
                    cs[l].copy_(c)
        # (5) replay, LSTM state written back as the eager path leaves it (the rows of the last output length)
        G.graph.replay()
        r0 = 0 if lens is None else order.index(len(lens) - 1) * grows
        r1 = r0 + (rows if lens is None else grows)
        for m in ("posterior", "prior", "frame_predictor"):
            hs, cs = G.bufs[f"{m}_h"], G.bufs[f"{m}_c"]
            getattr(model, m).hidden = [(hs[l, r0:r1].clone(), cs[l, r0:r1].clone()) for l in range(hs.shape[0])]
        return G, slots

    def _assemble(self, G, x, slots, len_output):
        """Steps (6)-(7) of a one-segment call: the generated sequence (or nsample sequences) as fresh tensors out of the
        graph's buffers."""
        return self._assemble_seq(G.cfg, G.bufs["out"].clone(), x, slots, len_output)

    def _assemble_seq(self, c, out, x, slots, len_output):
        """The returned list of one segment from its decoded frames out (already out of graph memory): ground truth while
        i < n_past, zeros for skipped frames."""
        nsample, B, n_past, fshape, dev, rows = c["ns"], c["B"], c["n_past"], c["fshape"], c["dev"], c["rows"]
        executed = {i for (i, _, _, _) in slots}
        frames, j = [], 0
        for i in range(1, len_output):
            if i not in executed:
                frames.append(None)
            elif i < n_past:
                frames.append(x[i])
            else:
                frames.append(out[j])
                j += 1
        seq = [x[0]] + frames
        zeros = torch.zeros((rows, *fshape), device=dev, dtype=x[0].dtype)
        if nsample == 1:
            return [f if f is not None else zeros.clone() for f in seq]
        res = [[] for _ in range(nsample)]
        for i, f in enumerate(seq):
            if f is None:
                f = zeros.clone()
            elif i == 0 or i < n_past:
                f = f.repeat(nsample, *([1] * (f.dim() - 1)))
            for s in range(nsample):
                res[s].append(f[s * B:(s + 1) * B])
        return res

    # ------------------------------------------------------------------ backbone hooks
    def _check_model(self):
        check_supported(self.model)

    def _frame_shape(self, f):
        """The per-row shape of an input frame; ValueError when the backbone cannot take it."""
        enc = self.model.encoder
        if f.dim() != 4 or tuple(f.shape[1:]) != (enc.nc, enc.image_width, enc.image_width):
            raise ValueError(f"frames of shape {tuple(f.shape)} do not fit the {enc.image_width}-pixel, {enc.nc}-channel backbone")
        return tuple(int(v) for v in f.shape[1:])

    def memory_bytes(self):
        """Device memory held by the cached graphs' buffers (the graphs' private pools come on top)."""
        return sum(t.numel() * t.element_size() for G in self._graphs.values() for t in G.bufs.values())

    def clear(self):
        """Drop every cached graph and its buffers.  The body keeps the graph it last ran in self.G (and its backend in
        self.K) for the layer helpers; those references go too, or the last graph's buffers would outlive the call."""
        self._graphs.clear()
        self.K = self.G = None

    # ------------------------------------------------------------------ buffers
    def _alloc_io(self, G):
        c, model = G.cfg, self.model
        dev, S, rows = c["dev"], c["S"], c["rows"]
        b = G.bufs
        b["x"] = torch.zeros(c["T_enc"] * c["B"], *c["fshape"], device=dev)
        b["tab_int"] = torch.zeros(max(4 * S, 1), dtype=torch.int32, device=dev)
        b["tab_f"] = torch.zeros(max(2 * S * c["nG"], 1), device=dev)
        b["eps"] = torch.zeros(max(S, 1), 2, rows, model.z_dim, device=dev)
        n_dec = c["n_dec"]
        b["out"] = torch.zeros(max(n_dec, 1), rows, *c["fshape"], device=dev)[:n_dec]
        for m in ("posterior", "prior", "frame_predictor"):
            mod = getattr(model, m)
            for k in ("h", "c"):
                b[f"{m}_{k}"] = torch.zeros(mod.n_layers, rows, mod.hidden_size, device=dev)   # updated in place by the graph

    def _buf(self, G, name, numel, dtype=torch.float32):
        """Buffer `name` of numel elements.  With several output lengths (generate_lengths) a request may be a prefix of the
        buffer: it is allocated at its first request, which is its largest, as the active row count of the steps never grows
        (plan_lengths)."""
        t = G.bufs.get(name)
        if t is None:
            t = G.bufs[name] = torch.zeros(int(numel), dtype=dtype, device=G.cfg["dev"])
        assert t.dtype == dtype and (t.numel() == numel or (G.cfg["nG"] > 1 and t.numel() > numel)), name
        return t if t.numel() == numel else t[:numel]

    # ------------------------------------------------------------------ the captured sequence
    def _body(self, G):
        from . import infer
        c, model = G.cfg, self.model
        K = infer.kernels_for(c["dev"])
        self.K, self.G = K, G
        rows, B, T, S, segs = c["rows"], c["B"], c["T"], c["S"], c["segs"]
        g, z = model.g_dim, model.z_dim
        nK = len(segs)
        self._prepare_weights()
        # ground truth: one time-batched encode at B rows (the clip, then a chain's skip-source copies), tiled to the
        # nsample*B rows of the recurrent part
        N = c["T_enc"] * B
        h_gt = self._buf(G, "gt_h", N * g)
        gt_skips = self._encode("gt", G.bufs["x"], N, h_gt)
        hsrc = {}

        def Hsrc(M):
            """[T + 1][M][g] for a step on M rows: the ground truth frames, then this step's h (the module input tables
            index rows with stride M)"""
            t = hsrc.get(M)
            if t is None:
                t = hsrc[M] = self._buf(G, "Hsrc" if M == rows else f"Hsrc{M}", (T + 1) * M * g)
                K.permute4(h_gt, t, (T, M // B, B * g, 1), (B * g, 0, 1, 0))
            return t

        Hsrc(rows)
        self._buf(G, "grp_zero", max(rows // B, 1), torch.int32)   # source image n % B for every sample

        # the skip sources of all segments: one frame in place (one segment), or the nK copies behind the clip (a chain)
        f0 = c["src"][0] if nK == 1 else T
        src_skips = [s[f0 * B * s.numel() // N:(f0 + nK) * B * s.numel() // N] for s in gt_skips]
        halves0 = None
        if any(Sk > n_tf for (_, _, _, Sk, n_tf) in segs) and not c["lfs"]:
            # models/p2p_model.py:143-144: the last skip set while i == 1 or i < n_past comes from x_k[max(n_past - 2, 0)]
            halves0 = self._skip_halves("skip", src_skips, nK * B)
        ti, tf = G.bufs["tab_int"], G.bufs["tab_f"]
        nG, active = c["nG"], c["active"]
        cr = c["grows"] if nG > 1 else 0   # rows per counter group (one group: the counters apply to every row)
        zbuf = self._buf(G, "Z", 2 * rows * z)
        h_pred = self._buf(G, "h_pred", rows * g)
        eps = G.bufs["eps"]
        s, d = 0, 0   # chain slot, decoded frame
        for k, (_, _, _, Sk, n_tf) in enumerate(segs):
            prev_frame = None
            for j in range(Sk):
                M = active[s]   # the rows still generating: a prefix
                Hs = Hsrc(M)
                zb = zbuf[:2 * M * z]
                tuc, dt = tf[s * nG:(s + 1) * nG], tf[(S + s) * nG:(S + s + 1) * nG]
                skips_cur = None
                if j > n_tf:   # the previous step's decoded frame: the only autoregressive encoder call
                    skips_cur = self._encode("step", prev_frame, M, Hs[T * M * g:])
                glob = ti[3 * S + s:3 * S + s + 1]
                # posterior || prior in one launch, then the frame predictor (models/p2p_model.py:150-179)
                K.lstm_step([self._module("posterior", Hs, ti[s:s + 1], Hs, glob, g, tuc, dt, cr, eps=eps[s, 0], out=zb[:M * z]),
                             self._module("prior", Hs, ti[S + s:S + s + 1], Hs, glob, g, tuc, dt, cr, eps=eps[s, 1],
                                          out=zb[M * z:])], M, model.rnn_size)
                K.lstm_step([self._module("frame_predictor", Hs, ti[S + s:S + s + 1], zb, ti[2 * S + s:2 * S + s + 1], z, tuc,
                                          dt, cr, out=h_pred)], M, model.rnn_size)
                s += 1
                if j < n_tf:
                    continue   # teacher-forced step: the predictor only advances its state (models/p2p_model.py:157-163)
                if c["lfs"] and j > n_tf:
                    halves = self._skip_halves("skip", skips_cur, M)
                else:
                    if halves0 is None:   # last_frame_skip: every segment's first decode, batched at the chain's first
                        halves0 = self._skip_halves("skip0", src_skips, nK * B)
                    halves = self._segment_halves(halves0, k, nK)
                prev_frame = G.bufs["out"][d]
                d += 1
                self._decode(h_pred, halves, prev_frame, M)

    def _segment_halves(self, halves, k, nK):
        """Segment k's part of skip halves computed for the nK segments' sources at once (B images each)."""
        if nK == 1:
            return halves
        return [(t[k * t.numel() // nK:(k + 1) * t.numel() // nK], nsrc // nK) for t, nsrc in halves]

    # ------------------------------------------------------------------ weights
    def _prepare_weights(self):
        from . import infer
        K, G, model = self.K, self.G, self.model
        adt = G.cfg["adt"]
        enc, dec = model.encoder, model.decoder
        self.chans = infer._stages(enc)
        n = len(self.chans)
        self.wp, self.bn = {}, {}
        cin = enc.nc
        for l in range(n):
            conv, bn = getattr(enc, f"c{l + 1}").main[:2]
            cout = conv.weight.shape[0]
            wp = self._buf(G, f"wp_enc{l}", cout * 16 * cin, adt)
            pack_conv4(K, conv.weight.data, wp)
            self.wp[f"enc{l}"] = wp
            self._bn_coeffs(f"enc{l}", bn)
            cin = cout
        self._prepare_latent(getattr(enc, f"c{n + 1}"), dec.upc1)
        for k in range(n):
            last = k == n - 1
            blk = getattr(dec, f"upc{k + 2}")
            convt = blk[0] if last else blk.main[0]
            ci2, cout = convt.weight.shape[0], convt.weight.shape[1]
            wp = self._buf(G, f"wp_dec{k}", ci2 * 16 * cout, adt)
            pack_convt4(K, convt.weight.data, wp)
            self.wp[f"dec{k}"] = wp
            if not last:
                self._bn_coeffs(f"dec{k}", blk.main[1])

    def _bn_coeffs(self, tag, bn):
        """Eval-mode scale / shift of BatchNorm module bn from its running statistics, into self.bn[tag]."""
        G, C = self.G, bn.weight.numel()
        sc, sh = self._buf(G, f"bn_{tag}_scale", C), self._buf(G, f"bn_{tag}_shift", C)
        self.K.bn_eval_coeffs(bn.weight.data, bn.bias.data, bn.running_mean, bn.running_var, C, sc, sh, eps=bn.eps)
        self.bn[tag] = (sc, sh)

    def _prepare_latent(self, top, upc1):
        """Weights and eval-BatchNorm coefficients of the two latent layers both image backbones share: the encoder's top
        ``top`` = Conv2d(512, g, 4, 1, 0) + BatchNorm + Tanh and the decoder's head ``upc1`` = ConvTranspose2d(g, 512, 4, 1, 0) +
        BatchNorm + LeakyReLU."""
        K, G, g = self.K, self.G, self.model.g_dim
        adt = G.cfg["adt"]
        wp = self._buf(G, "wp_enc_top", g * 16 * 512, adt)
        pack_conv4(K, top[0].weight.data, wp)
        self.wp["enc_top"] = wp
        self._bn_coeffs("enc_top", top[1])
        wp = self._buf(G, "wp_dec-1", g * 16 * 512, adt)
        pack_convt4(K, upc1[0].weight.data, wp)
        b16 = self._buf(G, "bias16_dec-1", 16 * 512)
        tile_bias(K, upc1[0].bias.data, b16, 16)
        self.wp["dec-1"], self.wp["dec-1.bias16"] = wp, b16
        self._bn_coeffs("dec-1", upc1[1])

    # ------------------------------------------------------------------ encoder / decoder
    def _encode(self, tag, frames, N, h_out):
        """frames: fp32 NCHW [N, nc, W, W] -> h_out fp32 [N, g]; returns the skip maps (NHWC)."""
        K, G, model = self.K, self.G, self.model
        adt = G.cfg["adt"]
        enc = model.encoder
        H, cin = G.cfg["W"], enc.nc
        a = self._buf(G, f"{tag}_in", N * H * H * cin, adt)
        nchw_to_nhwc(K, frames, a, N, H * H, cin)
        skips = []
        for l, cout in enumerate(self.chans):
            conv = getattr(enc, f"c{l + 1}").main[0]
            Ho = H // 2
            M = N * Ho * Ho
            sc, sh = self.bn[f"enc{l}"]
            y = self._buf(G, f"{tag}_enc_y{l}", M * cout, adt)
            if adt == torch.bfloat16 and implicit_shape(cin, cout):
                K.conv_gemm(0, a, self.wp[f"enc{l}"], y, N, Ho, Ho, cin, cout, bias=conv.bias.data, eval_scale=sc, eval_shift=sh,
                            act=ACT_LRELU)
            else:
                col = self._buf(G, f"{tag}_enc_col{l}", M * 16 * cin, adt)
                raw = self._buf(G, f"{tag}_enc_raw{l}", M * cout, adt)
                K.im2col(a, col, N, H, H, cin)
                K.gemm(col, self.wp[f"enc{l}"], raw, M, cout, 16 * cin, bias=conv.bias.data)
                K.bn_act(raw, y, sc, sh, 1, M, cout, ACT_LRELU)
            skips.append(y)
            a, H, cin = y, Ho, cout
        self._encode_top(tag, a, N, h_out, getattr(enc, f"c{len(self.chans) + 1}")[0].bias)
        return skips

    def _encode_top(self, tag, a, N, h_out, bias):
        """The encoder's top layer (bias: its conv bias) on the 4x4x512 maps a [N, 4, 4, 512] -> h_out fp32 [N, g]."""
        K, G, g = self.K, self.G, self.model.g_dim
        adt = G.cfg["adt"]
        sc, sh = self.bn["enc_top"]
        raw = self._buf(G, f"{tag}_enc_rawf", N * g, adt)
        y = h_out if adt == torch.float32 else self._buf(G, f"{tag}_enc_yf", N * g, adt)
        K.gemm(a, self.wp["enc_top"], raw, N, g, 16 * 512, bias=bias.data)
        K.bn_act(raw, y, sc, sh, 1, N, g, ACT_TANH)
        if y is not h_out:
            cast(K, y, h_out, N * g)

    def _skip_halves(self, tag, skips, nsrc):
        """The skip half of every decoder stage's torch.cat([d, skip]) ConvTranspose for one skip source of nsrc images:
        implicit stages get the bias-free kind-2 product (added in the main GEMM's epilogue), explicit stages the tap
        products col2 of p2pvg_col2im_k4s2p1.  Returns per stage (tensor, imgs_per_group) for the decodes."""
        K, G = self.K, self.G
        adt = G.cfg["adt"]
        n = len(self.chans)
        out = []
        Hi = 4
        for k in range(n):
            cd = self.chans[n - 1 - k]
            cout = self.model.decoder.nc if k == n - 1 else self.chans[n - 2 - k]
            wS = self.wp[f"dec{k}"][cd * 16 * cout:]
            sk = skips[n - 1 - k]
            if adt == torch.bfloat16 and implicit_shape(cd, cout) and k < n - 1:
                addS = self._buf(G, f"{tag}_addS{k}", nsrc * 4 * Hi * Hi * cout, adt)
                K.conv_gemm(2, sk, wS, addS, nsrc, Hi, Hi, cd, cout)
            else:
                addS = self._buf(G, f"{tag}_colS{k}", nsrc * Hi * Hi * 16 * cout, adt)
                K.gemm(sk, wS, addS, nsrc * Hi * Hi, 16 * cout, cd, b_mn=True)
            out.append((addS, nsrc))
            Hi *= 2
        return out

    def _decode(self, h_pred, halves, frame_out, rows):
        """h_pred fp32 [rows, g] -> frame_out fp32 NCHW [rows, nc, W, W] (sigmoid applied), on the first rows rows."""
        K, G, model = self.K, self.G, self.model
        adt = G.cfg["adt"]
        dec = model.decoder
        n = len(self.chans)
        d = self._buf(G, "dec_d-1", rows * 16 * 512, adt)
        self._decode_head(h_pred, rows, self._buf(G, "dec_raw-1", rows * 16 * 512, adt), d)
        Hi = 4
        for k in range(n):
            last = k == n - 1
            cd = self.chans[n - 1 - k]
            cout = dec.nc if last else self.chans[n - 2 - k]
            blk = getattr(dec, f"upc{k + 2}")
            convt = blk[0] if last else blk.main[0]
            wD = self.wp[f"dec{k}"][:cd * 16 * cout]
            addS, nsrc = halves[k]
            gsrc = self.G.bufs["grp_zero"]
            Mo = rows * 4 * Hi * Hi
            y = self._buf(G, f"dec_y{k}", Mo * cout, adt)
            if adt == torch.bfloat16 and implicit_shape(cd, cout) and not last:
                sc, sh = self.bn[f"dec{k}"]
                K.conv_gemm(2, d, wD, y, rows, Hi, Hi, cd, cout, bias=convt.bias.data, addend=addS, grp_src=gsrc,
                            imgs_per_group=nsrc, eval_scale=sc, eval_shift=sh, act=ACT_LRELU)
            else:
                colD = self._buf(G, f"dec_colD{k}", rows * Hi * Hi * 16 * cout, adt)
                K.gemm(d, wD, colD, rows * Hi * Hi, 16 * cout, cd, b_mn=True)
                raw = y if last else self._buf(G, f"dec_raw{k}", Mo * cout, adt)
                K.col2im(colD, raw, rows, Hi, Hi, cout, bias=convt.bias.data, col2=addS, grp_src=gsrc, imgs_per_group=nsrc)
                if not last:
                    sc, sh = self.bn[f"dec{k}"]
                    K.bn_act(raw, y, sc, sh, 1, Mo, cout, ACT_LRELU)
            d = y
            Hi *= 2
        W, nc = Hi, dec.nc
        out32 = self._buf(G, "dec_out32", rows * W * W * nc)
        cast(K, d, out32, rows * W * W * nc)
        K.act_fwd(out32, out32.numel(), ACT_SIGMOID)
        nhwc_to_nchw(K, out32, frame_out, rows, W * W, nc)

    def _decode_head(self, h_pred, rows, raw, d):
        """The decoder's head upc1 on the first rows rows of h_pred fp32 [rows, g] -> d [rows, 4, 4, 512] (raw: its
        pre-BatchNorm scratch of the same size)."""
        K, G, g = self.K, self.G, self.model.g_dim
        adt = G.cfg["adt"]
        if adt == torch.float32:
            hp = h_pred
        else:
            hp = self._buf(G, "dec_hp", rows * g, adt)
            cast(K, h_pred, hp, rows * g)
        K.gemm(hp, self.wp["dec-1"], raw, rows, 16 * 512, g, b_mn=True, bias=self.wp["dec-1.bias16"])
        sc, sh = self.bn["dec-1"]
        K.bn_act(raw, d, sc, sh, 1, rows * 16, 512, ACT_LRELU)

    # ------------------------------------------------------------------ recurrent modules
    def _module(self, m, seg_a, idx_a, seg_b, idx_b, gb, tuc, dt, counter_rows, eps=None, out=None):
        """p2pvg_lstm_step operands of module m for one step: input [seg_a[idx_a] | seg_b[idx_b] | tuc | dt], state updated in
        place in the graph's [L][rows][R] buffers, gaussian head (with eps) or Linear + tanh head; counter_rows > 0: row b
        reads the counters tuc[b / counter_rows], dt[b / counter_rows]."""
        from ._lib import LSTM_HEAD_GAUSSIAN, LSTM_HEAD_LINEAR_TANH
        G, mod = self.G, getattr(self.model, m)
        dev = G.cfg["dev"]
        tabs = G.bufs.get(f"{m}_ptrs")
        if tabs is None:   # device tables of pointers (the parameter addresses are part of the graph's signature)
            hs, cs = G.bufs[f"{m}_h"], G.bufs[f"{m}_c"]
            w = [t.data_ptr() for c in mod.lstm for t in (c.weight_ih, c.bias_ih, c.weight_hh, c.bias_hh)]
            st = [t.data_ptr() for l in range(mod.n_layers) for t in (hs[l], cs[l], hs[l], cs[l])]
            tabs = G.bufs[f"{m}_ptrs"] = torch.tensor(w + st, dtype=torch.int64, device=dev)
        L = mod.n_layers
        d = dict(seg_a=seg_a, idx_a=idx_a, ga=self.model.g_dim, seg_b=seg_b, idx_b=idx_b, gb=gb, tuc=tuc, dt=dt, counter_rows=counter_rows,
                 w_embed=mod.embed.weight, b_embed=mod.embed.bias, layers=L, layer_w=tabs[:4 * L], state=tabs[4 * L:], out=out)
        if hasattr(mod, "mu_net"):
            d.update(head=LSTM_HEAD_GAUSSIAN, out_dim=mod.output_size, w_out=mod.mu_net.weight, b_out=mod.mu_net.bias,
                     w_out2=mod.logvar_net.weight, b_out2=mod.logvar_net.bias, eps=eps)
        else:
            d.update(head=LSTM_HEAD_LINEAR_TANH, out_dim=mod.output_size, w_out=mod.output[0].weight, b_out=mod.output[0].bias)
        return d


class PoseGenerateEngine(GenerateEngine):
    """p2p_generate_graphed for the h36m_mlp pose backbone (models/h36m_mlp.py): the planner, tables, eps, LSTM state and
    output assembly of GenerateEngine; every encoder and decoder call is ONE p2pvg_pose_mlp launch reading the live
    parameters (exact fp32 in both P2PVG_PRECISION modes, as the eager pose path).  The ground-truth encode keeps its skips
    h1 / h2 at B rows; the decoder reads skip row r % B for output row r."""

    def _check_model(self):
        check_supported_pose(self.model)

    def _frame_shape(self, f):
        if f.dim() != 3 or tuple(f.shape[1:]) != (17, 3):
            raise ValueError(f"p2p_generate_graphed takes [B, 17, 3] poses for the h36m_mlp backbone (got frames of shape "
                             f"{tuple(f.shape)}); use p2p_generate")
        return (17, 3)

    def _prepare_weights(self):
        pass   # the kernel reads the parameters in place; their addresses are part of the graph's signature

    def vis_canvas(self, *args, **kwargs):
        raise ValueError("poses are rendered on the host before they are composed: p2pvg_b200.visualize.vis_seq composes "
                         "the uploaded images")

    def _encode(self, tag, frames, N, h_out):
        G, g = self.G, self.model.g_dim
        h1, h2 = self._buf(G, f"{tag}_h1", N * g), self._buf(G, f"{tag}_h2", N * g)
        self.K.pose_mlp(self.model.encoder, False, frames, h_out, N, h1=h1, h2=h2)
        return [h1, h2]

    def _skip_halves(self, tag, skips, nsrc):
        return skips, nsrc

    def _segment_halves(self, halves, k, nK):
        skips, nsrc = halves
        if nK == 1:
            return halves
        return [s[k * s.numel() // nK:(k + 1) * s.numel() // nK] for s in skips], nsrc // nK

    def _decode(self, h_pred, halves, frame_out, rows):
        skips, nsrc = halves
        self.K.pose_mlp(self.model.decoder, True, h_pred, frame_out, rows, skips=skips, nsrc=nsrc)
