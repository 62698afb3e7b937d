"""``models.p2p_model.P2PModel`` drop-in (reference models/p2p_model.py:12-330): same constructor, attributes
(``encoder``, ``decoder``, ``frame_predictor``, ``posterior``, ``prior``, ``*_optimizer``), ``forward`` return
value, ``save`` / ``load`` checkpoint format — with ``forward`` executed by p2pvg_b200.engine.TrainEngine on
hand-written sm_90a kernels.  ``train.py`` / ``generate.py`` of the reference run against it unchanged.

Differences that are visible and documented (DESIGN.md): after ``forward`` the ``.grad`` of the four non-prior
modules holds the gradient that was *applied* (backward #1); the reference additionally accumulates the
never-applied backward #2 contribution there (SURVEY.md A.3 item 11).
"""
import math
import os

import numpy as np
import torch
import torch.nn as nn

from . import lstm as lstm_models
from ..misc import criterion, utils

MODULES = ("frame_predictor", "posterior", "prior", "encoder", "decoder")


class ArenaAdam(torch.optim.Optimizer):
    """``torch.optim.Adam``-shaped handle (state_dict layout: step / exp_avg / exp_avg_sq per parameter) over one
    module's flat parameter arena.  The update itself is the fused kernel p2pvg_adam_legacy, launched by the
    engine inside the train step (PyTorch-1.0 arithmetic, which is what the reference pins)."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8):
        # the param_groups carry every key stock torch.optim.Adam reads in step(), so that a checkpoint written here
        # resumes under the reference's real optim.Adam (Adam.load_state_dict replaces its param_groups with the saved ones)
        super().__init__(list(params), dict(lr=lr, betas=betas, eps=eps, weight_decay=0, amsgrad=False, maximize=False,
                                            foreach=None, capturable=False, differentiable=False, fused=None,
                                            decoupled_weight_decay=False))
        self._arena = None
        self._names = None

    def attach(self, arena, named_params):
        self._arena = arena
        for name, p in named_params:
            m, v = arena.moment_views(name)
            old = self.state.get(p, {})
            if "exp_avg" in old:
                m.copy_(old["exp_avg"])
                v.copy_(old["exp_avg_sq"])
                arena.step_t.fill_(int(old.get("step", 0)))
            self.state[p] = dict(step=int(arena.step_t.item()), exp_avg=m, exp_avg_sq=v)

    def sync_step(self):
        if self._arena is not None:
            t = int(self._arena.step_t.item())
            for st in self.state.values():
                st["step"] = t

    def state_dict(self):
        self.sync_step()
        return super().state_dict()

    def load_state_dict(self, sd):
        arena = self._arena
        super().load_state_dict(sd)
        for g in self.param_groups:   # checkpoints of older optimisers (e.g. PyTorch 1.0 Adam) lack newer hyper-parameter keys
            for k, v in self.defaults.items():
                g.setdefault(k, v)
        if arena is not None:  # re-home the loaded moments into the arena views
            names = {id(p): n for n, p in self._named}
            for p, st in list(self.state.items()):
                m, v = arena.moment_views(names[id(p)])
                m.copy_(st["exp_avg"])
                v.copy_(st["exp_avg_sq"])
                arena.step_t.fill_(int(st["step"]))
                self.state[p] = dict(step=int(st["step"]), exp_avg=m, exp_avg_sq=v)

    def step(self, closure=None):
        raise RuntimeError("ArenaAdam.step() is fused into P2PModel.forward (the reference also steps inside forward)")


class P2PModel(nn.Module):
    def __init__(self, batch_size=100, channels=1, g_dim=128, z_dim=10, rnn_size=256, prior_rnn_layers=1,
                 posterior_rnn_layers=1, predictor_rnn_layers=2, opt=None):
        super().__init__()
        self.batch_size, self.channels, self.g_dim, self.z_dim, self.rnn_size = batch_size, channels, g_dim, z_dim, rnn_size
        self.prior_rnn_layers, self.posterior_rnn_layers, self.predictor_rnn_layers = prior_rnn_layers, posterior_rnn_layers, predictor_rnn_layers
        self.opt = opt
        # construction order == reference (p2p_model.py:28-38) so the torch RNG stream matches
        self.frame_predictor = lstm_models.lstm(g_dim + z_dim + 2, g_dim, rnn_size, predictor_rnn_layers, batch_size)
        self.posterior = lstm_models.gaussian_lstm(2 * g_dim + 2, z_dim, rnn_size, posterior_rnn_layers, batch_size)
        self.prior = lstm_models.gaussian_lstm(2 * g_dim + 2, z_dim, rnn_size, prior_rnn_layers, batch_size)
        self.is_pose = getattr(opt, "dataset", None) == "h36m"
        if self.is_pose:  # models/p2p_model.py:33-35
            self.encoder = opt.backbone_net.encoder(out_dim=g_dim, h_dim=g_dim)
            self.decoder = opt.backbone_net.decoder(in_dim=g_dim, h_dim=g_dim)
        else:
            self.encoder = opt.backbone_net.encoder(g_dim, channels)
            self.decoder = opt.backbone_net.decoder(g_dim, channels)
        opt.optimizer = ArenaAdam
        self.mse_criterion = nn.MSELoss()
        self.kl_criterion = criterion.KLCriterion(opt=opt)
        self.align_criterion = nn.MSELoss()
        self._engine = None
        self.precision = os.environ.get("P2PVG_PRECISION", "bf16")
        self.use_graph = os.environ.get("P2PVG_GRAPH", "1") != "0"
        self.update_mode = os.environ.get("P2PVG_UPDATE_MODE", "A")
        self.init_weight()
        self.init_optimizer()

    # ---- reference API -----------------------------------------------------------------------------
    def init_optimizer(self):
        opt = self.opt
        for m in MODULES:
            o = opt.optimizer(getattr(self, m).parameters(), lr=opt.lr, betas=(opt.beta1, 0.999))
            o._named = list(getattr(self, m).named_parameters())
            setattr(self, m + "_optimizer", o)
        self._engine = None

    def init_hidden(self, batch_size=1):
        self.frame_predictor.hidden = self.frame_predictor.init_hidden(batch_size=batch_size)
        self.posterior.hidden = self.posterior.init_hidden(batch_size=batch_size)
        self.prior.hidden = self.prior.init_hidden(batch_size=batch_size)

    def init_weight(self):
        for m in MODULES:
            getattr(self, m).apply(utils.init_weights)

    def get_global_descriptor(self, x, start_ix=0, cp_ix=None):
        if cp_ix is None:
            cp_ix = len(x) - 1
        x_cp = x[cp_ix]
        return x_cp, self.encoder(x_cp)[0]

    # ---- engine binding ----------------------------------------------------------------------------
    def _opt_dict(self):
        o = self.opt
        return dict(beta=float(o.beta), weight_cpc=float(o.weight_cpc), weight_align=float(o.weight_align),
                    skip_prob=float(o.skip_prob), n_past=int(o.n_past), last_frame_skip=bool(o.last_frame_skip),
                    lr=float(o.lr), beta1=float(o.beta1), batch_size=int(o.batch_size))

    def engine(self, width):
        if self._engine is not None:
            return self._engine
        from .._lib import kernels_for
        from ..engine import TrainEngine
        from ..engine_mlp import TrainEngineMLP
        from ..engine_vgg import TrainEngineVGG
        dev = next(self.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("p2pvg_b200 has no CPU path: move the model to a CUDA device first (model.cuda())")
        cfg = dict(g_dim=self.g_dim, z_dim=self.z_dim, rnn_size=self.rnn_size, channels=self.channels, image_width=width,
                   backbone="mlp" if self.is_pose else getattr(self.encoder, "backbone", "dcgan"))
        state = {m: getattr(self, m).state_dict() for m in MODULES}
        adt = torch.float32 if self.precision == "fp32" else torch.bfloat16
        cls = {"mlp": TrainEngineMLP, "vgg": TrainEngineVGG}.get(cfg["backbone"], TrainEngine)
        eng = cls(state, cfg, self._opt_dict(), kernels_for(dev), act_dtype=adt, mode=self.update_mode)
        self._grad_views = []
        for m in MODULES:
            mod = getattr(self, m)
            named = list(mod.named_parameters())
            for k, p in named:  # parameters become views of the flat arena; .grad views of the grad arena
                p.data = eng.arena[m].p[k]
                p.grad = eng.arena[m].g[k]
            for k in list(eng.buffers[m].keys()):
                owner, _, leaf = k.rpartition(".")
                mod.get_submodule(owner)._buffers[leaf] = eng.buffers[m][k]
            getattr(self, m + "_optimizer").attach(eng.arena[m], named)
            self._grad_views += [(p, eng.arena[m].g[k]) for k, p in named]
        self._engine = eng
        return eng

    def forward(self, x, start_ix=0, cp_ix=-1):
        """One training step; returns (mse, kld, cpc, align) numpy scalars divided by seq_len
        (reference models/p2p_model.py:185-271)."""
        if isinstance(x, tuple):  # h36m: (pose_2d, pose_3d, camera_view) -> pose_3d (models/p2p_model.py:187-189)
            x = x[1]
        if not torch.is_tensor(x):
            x = torch.stack(list(x))
        eng = self.engine(int(x.shape[-1]))
        eng.opt = self._opt_dict()
        out = eng.step(x.float(), use_graph=self.use_graph, return_device=True)
        # model.zero_grad() drops .grad; keep them readable for train.py's histograms.  The views are static, so this host work
        # is done while the GPU runs the step, BEFORE the blocking read-back of the four scalars
        for p, g in self._grad_views:
            p.grad = g
        # the scalars are final after the forward half of the step: the engine hands them over as soon as they exist (zero-copy
        # store polled by the host) while the backward passes and the optimiser still run; any later use of the model is
        # stream-ordered behind them (P2PVG_EARLY_LOSS=0: blocking read-back after the whole step)
        host = eng.read_losses(out)
        return host[0], host[1], host[2], host[3]

    def p2p_losses(self, x):
        """The training objective on a held-out batch, without an update (an addition to the reference API): the four values
        forward(x) returns with every module in eval mode -- BatchNorm normalising with its running statistics -- computed
        before any update, with the same NumPy skip draw and the same torch.randn eps draw as forward, and nothing changed:
        parameters, .grad, Adam moments and steps and BatchNorm buffers stay bit-identical, and captured training graphs stay
        valid whatever the held-out batch's T, B and skip pattern (its buffers that the training step has not already
        sized come from a pool of their own).  One CUDA-graph replay per call
        (engine.TrainEngine.evaluate_losses, kernel p2pvg_seq_losses).

        x: what forward takes.  Returns a dict: 'mse', 'kld', 'cpc', 'align' (floats, / seq_len, KL / opt.batch_size),
        'per_sequence': per term a float64 [B] device tensor of each row's share (element means over row b for mse, cpc and
        align, whose row mean is the scalar; row b's KL sum / opt.batch_size for kld, whose row sum is the scalar), and
        'steps': the executed timesteps i of the skip schedule.  ValueError before any draw or launch for a model with a
        module in training mode, a model or x not on a CUDA device, or fewer than 2 frames."""
        for m in MODULES:
            if any(mod.training for mod in getattr(self, m).modules()):
                raise ValueError(f"p2p_losses needs every module in eval mode ({m} is in training mode); call model.eval() first")
        if isinstance(x, tuple):  # h36m: (pose_2d, pose_3d, camera_view) -> pose_3d, as forward
            x = x[1]
        if not torch.is_tensor(x):
            x = torch.stack(list(x))
        if x.dim() < 3 or int(x.shape[0]) < 2:
            raise ValueError(f"p2p_losses needs a [T, B, ...] batch with T >= 2 frames (got shape {tuple(x.shape)})")
        dev = next(self.parameters()).device
        if dev.type != "cuda" or not x.is_cuda:
            raise ValueError(f"p2p_losses runs on a CUDA device: the model is on {dev} and x on {x.device}; move both with .cuda()")
        eng = self.engine(int(x.shape[-1]))
        eng.opt = self._opt_dict()
        plan, per, out = eng.evaluate_losses(x.float(), use_graph=self.use_graph)
        host = out.cpu().numpy()
        names = ("mse", "kld", "cpc", "align")
        res = {k: float(host[j]) for j, k in enumerate(names)}
        res["per_sequence"] = {k: per[j] for j, k in enumerate(names)}
        res["steps"] = list(plan.tgt_frame)
        return res

    def p2p_generate(self, x, len_output, eval_cp_ix, start_ix=0, cp_ix=-1, model_mode='full', skip_frame=False,
                     init_hidden=True):
        from ..infer import p2p_generate
        return p2p_generate(self, x, len_output, eval_cp_ix, model_mode=model_mode, skip_frame=skip_frame, init_hidden=init_hidden)

    def p2p_generate_samples(self, x, nsample, len_output, eval_cp_ix, model_mode='full', skip_frame=False):
        """nsample samples per input sequence in one batched pass (an addition to the reference API; see infer.py)."""
        from ..infer import p2p_generate_samples
        return p2p_generate_samples(self, x, nsample, len_output, eval_cp_ix, model_mode=model_mode, skip_frame=skip_frame)

    def p2p_generate_graphed(self, x, len_output, eval_cp_ix, model_mode='full', skip_frame=False, init_hidden=True, nsample=1):
        """p2p_generate (nsample=1) or p2p_generate_samples (nsample>1) as one CUDA-graph replay per call (an addition to the
        reference API; see gen_engine.py and gen_engine_vgg.py).  dcgan_64 / dcgan_128, vgg_64 / vgg_128 (on a CUDA device)
        and h36m_mlp in eval mode only: anything else raises ValueError.  Pose input: the (pose_2d, pose_3d, camera_view)
        tuple, a [T, B, 17, 3] tensor or a list of [B, 17, 3]."""
        return self._graphed_engine().generate(x, len_output, eval_cp_ix, model_mode=model_mode, skip_frame=skip_frame,
                                               init_hidden=init_hidden, nsample=nsample)

    def p2p_generate_multi_cp(self, x, cp_ixs, len_outputs=None, model_mode='full', skip_frame=False, nsample=1):
        """Generation through several control points as ONE CUDA-graph replay (an addition to the reference API; see
        gen_engine.py).  Segment k is x_k = x[cp_ixs[k] : cp_ixs[k + 1] + 1], generated with L_k = len_outputs[k] frames
        (default: len(x_k), the clip's timing; any L_k >= 2).  The result is what the looped calls

            [p2p_generate_graphed(x_0, L_0, L_0 - 1, model_mode, skip_frame, init_hidden=True, nsample=nsample)] +
            [p2p_generate_graphed(x_k, L_k, L_k - 1, model_mode, skip_frame, init_hidden=False, nsample=nsample) for k >= 1]

        return -- a list of one such result per segment -- with the same NumPy draws (one per segment, in order), the same eps
        consumption under infer.eps_stream and the same final LSTM state in .hidden.  Segment k > 0 starts from its given
        control point x_k[0].  cp_ixs: strictly increasing ints, at least 2, cp_ixs[0] == 0, cp_ixs[-1] <= len(x) - 1; to
        generate from control points only pass the stacked control points and cp_ixs = range(K + 1).  x: what
        p2p_generate_graphed takes (for the pose tuple only pose_3d is read).  The same models as p2p_generate_graphed;
        ValueError before any launch for a malformed cp_ixs or len_outputs, or a segment shorter than min(n_past, L_k)."""
        return self._graphed_engine().generate_multi_cp(x, cp_ixs, len_outputs=len_outputs, model_mode=model_mode,
                                                        skip_frame=skip_frame, nsample=nsample)

    def p2p_generate_lengths(self, x, len_outputs, model_mode='full', nsample=1):
        """One start/end pair generated at several output lengths as ONE CUDA-graph replay (an addition to the reference API;
        see gen_engine.py).  Returns one result per entry of len_outputs, in order: what the looped calls

            [p2p_generate_graphed(x, L, L - 1, model_mode, skip_frame=False, nsample=nsample) for L in len_outputs]

        return, with the same NumPy draws (one per length, in order), the same eps consumption under infer.eps_stream and
        .hidden left holding the rows of len_outputs[-1].  The rows of every length share the replay: step i runs on the
        lengths greater than i only.  x: what p2p_generate_graphed takes.  The same models as p2p_generate_graphed;
        ValueError before any draw or launch for an empty or malformed len_outputs, a length below 2 or a length L with
        len(x) < min(n_past, L)."""
        return self._graphed_engine().generate_lengths(x, len_outputs, model_mode=model_mode, nsample=nsample)

    def p2p_evaluate(self, x, nsample=1, len_output=None, model_mode='full', data_range=1.0, cp_ixs=None):
        """Generate and score in one call (an addition to the reference API): exactly what
        p2p_generate_graphed(x, L, L - 1, model_mode, skip_frame=False, nsample=nsample) generates (same draws, same cached
        graph, .hidden left the same way), with L = len_output or len(x) (len(pose_3d) for the pose tuple), then ONE metrics
        launch (p2pvg_b200.metrics) on the generated frames.  Scored: every generated frame n_past .. L - 1 against x[i] when
        L == len(x), else only the control point L - 1 against x[len(x) - 1].  The same models as p2p_generate_graphed.

        cp_ixs: score a generation through control points instead -- exactly what p2p_generate_multi_cp(x, cp_ixs,
        model_mode=model_mode, nsample=nsample) generates (the clip's timing, skip_frame=False) -- with every generated frame
        n_past .. T_k - 1 of every segment scored against x[cp_ixs[k] + i]; 'frames' then holds the sorted clip indices, which
        include every control point cp_ixs[1:].  ValueError with len_output, or when a segment has no more than n_past frames.

        Returns a dict: 'frames' (the scored indices), per metric a float64 [nsample, len(frames), B] tensor on the device --
        mse, psnr, ssim for frames (data_range: the frames' value range), mse, mpjpe for poses; the last frame column is the
        control point -- and 'best': per metric (index [B], curve [len(frames), B]) of the sample with the best mean over the
        scored frames (highest ssim / psnr, lowest mse / mpjpe; the first on ties).  ValueError when L <= n_past or
        data_range is not positive."""
        return self._graphed_engine().evaluate(x, nsample=nsample, len_output=len_output, model_mode=model_mode,
                                               data_range=data_range, cp_ixs=cp_ixs)

    def p2p_evaluate_lengths(self, x, len_outputs, nsample=1, model_mode='full', data_range=1.0):
        """Generate at several output lengths and score them in one call (an addition to the reference API): ONE
        p2p_generate_lengths replay (the same draws, row groups and .hidden afterwards) and ONE metrics launch over every
        length's rows.  Returns one dict per entry of len_outputs, in order, each what the looped call

            p2p_evaluate(x, nsample, len_output=L, model_mode=model_mode, data_range=data_range)

        returns: L == len(x) scores every generated frame, any other L only the control point.  The same models as
        p2p_generate_graphed.  ValueError before any draw or launch for what p2p_generate_lengths rejects, a length <= n_past
        or a data_range that is not positive."""
        return self._graphed_engine().evaluate_lengths(x, len_outputs, nsample=nsample, model_mode=model_mode,
                                                       data_range=data_range)

    def _graphed_engine(self):
        from ..gen_engine import GenerateEngine, PoseGenerateEngine
        from ..gen_engine_vgg import VggGenerateEngine
        from .vgg import VggEncoder
        if getattr(self, "_gen_engine", None) is None:
            cls = PoseGenerateEngine if self.is_pose else VggGenerateEngine if isinstance(self.encoder, VggEncoder) else GenerateEngine
            self._gen_engine = cls(self)
        return self._gen_engine

    # ---- checkpoints (same dict layout as reference p2p_model.py:289-330) --------------------------
    def save(self, fname, epoch):
        backbone_net, optimizer = self.opt.backbone_net, getattr(self.opt, "optimizer", None)
        self.opt.backbone_net, self.opt.optimizer = 0, 0
        states = {m: getattr(self, m).state_dict() for m in MODULES}
        states.update({m + "_opt": getattr(self, m + "_optimizer").state_dict() for m in MODULES})
        states.update(epoch=epoch, opt=self.opt)
        torch.save(states, fname)
        self.opt.backbone_net, self.opt.optimizer = backbone_net, optimizer

    def load(self, pth=None, states=None):
        if states is None:
            states = torch.load(pth, weights_only=False)
        for m in MODULES:
            getattr(self, m).load_state_dict(states[m])
            getattr(self, m + "_optimizer").load_state_dict(states[m + "_opt"])
        keep = (self.opt.backbone_net, getattr(self.opt, "optimizer", None))
        self.opt = states["opt"]
        self.opt.backbone_net, self.opt.optimizer = keep
        return states["epoch"] + 1
