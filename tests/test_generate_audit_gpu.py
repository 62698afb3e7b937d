"""The graphed generation's launches against float64, where they run: a real call of every backbone with its CUDA-graph
replay replaced by GenerateEngine._body run eagerly on tests/gen_audit.GenAudit, every launch checked on its own operands
(p2pvg_lstm_step, p2pvg_pose_mlp, bn_eval_coeffs and the folded eval BatchNorm against the module's formula, the eval
epilogues of conv_gemm kinds 0 / 2 / 3 with grp_src addends, the explicit lowering, the vgg thin ends, the layout copies and
casts, the closing sigmoid), and the audited call equal to a plain replay of the same call bit for bit.

Per backbone (and P2PVG_PRECISION mode for the image backbones) one model with perturbed running statistics (a few channels
with |running_mean| >= 100 sqrt(running_var)) runs:
  * p2p_generate_graphed, nsample 20, B 22 (440 rows: grp_zero tiling, nsrc = 22 < rows; multi-round eval epilogues);
  * p2p_generate_lengths with three lengths, nsample 20, B 22 (1320 rows: counter_rows > 0, active prefixes below the rows;
    vgg_128 in fp32 at nsample 10, see test_audit_generate_image);
  * nsample 3, B 7 (21 rows: a partial 8-row slab);
  * a two-segment chain with last_frame_skip off and on, n_past 1 and 2 (segment halves, teacher-forced steps).
The predictor has 2 layers (R 256 for images, 512 for poses).  Output lengths are kept short so that the float64 references
stay within time and memory.
"""
import gc
import types
import weakref

import pytest
import torch

from oracle import p2p_oracle as O
from tests.gen_audit import GenAudit, audited_call
from tests.launch_audit import memory_per_test  # noqa: F401  (fixture)
from tests.launch_audit import release
from tests.loss_ref import ACT_LRELU, ACT_SIGMOID, ACT_TANH
from tests.test_generate_engine_gpu import precision

pytestmark = pytest.mark.gpu

NS, BB = 20, 22   # evaluate.py's default nsample, the reference's default batch


def _perturb(state, seed):
    """Non-trivial running statistics, with channels 0 and 1 of every BatchNorm at |running_mean| = 120 sqrt(running_var)
    (variance 1, so that the layer does not amplify its input and the activations stay in range through the stack)."""
    g = torch.Generator().manual_seed(seed)
    for m in ("encoder", "decoder"):
        for k, v in state[m].items():
            if k.endswith("running_mean"):
                v.copy_(0.1 * torch.randn(v.shape, generator=g))
            elif k.endswith("running_var"):
                v.copy_(0.5 + torch.rand(v.shape, generator=g))
        for k, v in state[m].items():
            if k.endswith("running_var"):
                mean = state[m][k[:-len("running_var")] + "running_mean"]
                v[:2] = 1.0
                mean[:2] = torch.tensor([120.0, -120.0])
    return state


def image_model(backbone, W, nc):
    from p2pvg_b200.models import dcgan_64, dcgan_128, vgg_64, vgg_128
    from p2pvg_b200.models.p2p_model import P2PModel
    net = {("dcgan", 64): dcgan_64, ("dcgan", 128): dcgan_128, ("vgg", 64): vgg_64, ("vgg", 128): vgg_128}[(backbone, W)]
    cfg = dict(g_dim=128, z_dim=10, rnn_size=256, channels=nc, image_width=W, predictor_rnn_layers=2, posterior_rnn_layers=1,
               prior_rnn_layers=1)
    if backbone == "vgg":
        cfg.update(backbone="vgg", vgg_width=W)
    opt = types.SimpleNamespace(dataset="mnist", backbone_net=net, lr=1e-3, beta1=0.9, beta=1e-4, weight_cpc=100.0,
                                weight_align=0.5, skip_prob=0.5, n_past=1, last_frame_skip=False, batch_size=BB)
    model = P2PModel(BB, nc, 128, 10, 256, 1, 1, 2, opt=opt)
    state = _perturb(O.build_state(cfg, seed=5), 6)
    for m in O.MODULES:
        getattr(model, m).load_state_dict(state[m])
    return model.cuda().eval()


def pose_model():
    from p2pvg_b200.models import h36m_mlp
    from p2pvg_b200.models.p2p_model import P2PModel
    cfg = dict(g_dim=128, z_dim=10, rnn_size=512, backbone="mlp", predictor_rnn_layers=2, posterior_rnn_layers=1, prior_rnn_layers=1)
    opt = types.SimpleNamespace(dataset="h36m", backbone_net=h36m_mlp, lr=1e-3, beta1=0.9, beta=1e-4, weight_cpc=100.0,
                                weight_align=0.5, skip_prob=0.5, n_past=1, last_frame_skip=False, batch_size=BB)
    model = P2PModel(BB, 1, 128, 10, 512, 1, 1, 2, opt=opt)
    state = O.build_state(cfg, seed=5)
    g = torch.Generator().manual_seed(6)
    for m in O.MODULES:   # weights moved off the N(0, 0.02) initialisation, as test_pose_generate_gpu.perturbed_state
        for v in state[m].values():
            if v.is_floating_point():
                v.add_(0.05 * torch.randn(v.shape, generator=g))
        getattr(model, m).load_state_dict(state[m])
    return model.cuda().eval()


def frames(T, B, shape, seed):
    g = torch.Generator().manual_seed(seed)
    if shape == (17, 3):
        return (3 * torch.randn(T, B, 17, 3, generator=g)).cuda()
    return torch.rand(T, B, *shape, generator=g).cuda()


def calls(shape, ns_lengths=NS):
    """(label, n_past, last_frame_skip, call) of every case; each call's result is a (nested) list of tensors."""
    T = 4
    nl = ns_lengths * BB * 3
    big, small, chain = frames(T, BB, shape, 1), frames(T, 7, shape, 2), frames(5, 2, shape, 3)
    out = [("graphed ns20 B22 rows440", 1, False, lambda m: m.p2p_generate_graphed(big, 3, 2, nsample=NS)),
           (f"lengths (4,2,3) ns{ns_lengths} B22 rows{nl}", 1, False,
            lambda m: m.p2p_generate_lengths(big, [4, 2, 3], nsample=ns_lengths)),
           ("graphed ns3 B7 rows21", 1, False, lambda m: m.p2p_generate_graphed(small, 4, 3, skip_frame=True, nsample=3))]
    for n_past in (1, 2):
        for lfs in (False, True):
            out.append((f"chain [0,2,4] n_past={n_past} lfs={lfs} ns2 B2", n_past, lfs,
                        lambda m: m.p2p_generate_multi_cp(chain, [0, 2, 4], nsample=2)))
    return out


def run_cases(model, shape, label, ns_lengths=NS):
    audit = GenAudit("cuda")
    seen = set()
    for k, (name, n_past, lfs, call) in enumerate(calls(shape, ns_lengths)):
        model._graphed_engine().clear()   # one cached signature at a time: the 1320-row graphs are large
        gc.collect()                      # earlier models and their engines form reference cycles that hold graph memory
        release()
        model.opt.n_past, model.opt.last_frame_skip = n_past, lfs
        audit.log, audit.seen = [], set()
        audited_call(model, call, audit, seed=k + 3)
        worst = max((w for _, _, w in audit.log), default=0.0)
        print(f"[audit] {label} {name}: {len(audit.log)} launches checked, worst error/bound {worst:.3g}")
        seen |= audit.seen
    if audit.bn_of:
        print(f"[audit] {label}: folded eval BatchNorm against the module's formula: at most {audit.fold_worst:.3g} |gamma|")
    model._graphed_engine().clear()
    release()
    return seen


LSTM_VARIANTS = {("lstm_step", 1), ("lstm_step", 2), ("lstm_step", "counter_rows", False), ("lstm_step", "counter_rows", True),
                 ("lstm_step", "partial_slab"), ("lstm_step", "layers", 2), ("bn_eval_coeffs", True)}


def _missing(seen, want):
    return sorted(want - seen, key=str)


IMAGE = [("dcgan", 64, 1), ("dcgan", 128, 3), ("vgg", 64, 1), ("vgg", 128, 3)]


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
@pytest.mark.parametrize("backbone,W,nc", IMAGE, ids=[f"{b}{w}" for b, w, _ in IMAGE])
def test_audit_generate_image(backbone, W, nc, prec):
    # vgg_128 in fp32 lowers its 128x128 64-channel layers through a 9 * 64-column im2col buffer: 50 GB at 1320 rows, more
    # than an 80 GB card holds beside the audit, so its lengths case runs at nsample 10 (660 rows)
    ns_lengths = 10 if (backbone, W, prec) == ("vgg", 128, "fp32") else NS
    with precision(prec):
        model = image_model(backbone, W, nc)
        seen = run_cases(model, (nc, W, W), f"{backbone}_{W} {prec}", ns_lengths)
    want = set(LSTM_VARIANTS) | {("bn_act", ACT_TANH, "float32" if prec == "fp32" else "bfloat16"),
                                 ("bn_act", ACT_LRELU, "float32" if prec == "fp32" else "bfloat16"),
                                 ("permute4", "float32", "float32")}
    if prec == "bf16":
        want |= {("permute4", "float32", "bfloat16"), ("permute4", "bfloat16", "float32")}
    if backbone == "dcgan":
        want |= {("act_fwd", ACT_SIGMOID), ("im2col", nc), ("col2im", nc, True)}
        if prec == "bf16":
            want |= {("conv_gemm", 0, True, False), ("conv_gemm", 2, True, True), ("conv_gemm", 2, False, False)}
        else:
            want |= {("col2im", 64, True), ("im2col", 64)}
    else:
        want |= {("vgg_first_eval", nc), ("vgg_last_eval", nc), ("maxpool2_fwd",), ("upsample2_fwd",)}
        if prec == "bf16":
            want |= {("conv_gemm", 3, True, True), ("conv_gemm", 3, True, False), ("conv_gemm", 3, False, False)}
        else:
            want |= {("gather_add",)}
    assert not _missing(seen, want), f"launch variants that did not occur: {_missing(seen, want)}"


def test_audit_generate_pose():
    model = pose_model()
    seen = run_cases(model, (17, 3), "h36m_mlp")
    want = (set(LSTM_VARIANTS) - {("bn_eval_coeffs", True)}) | {("pose_mlp", "encoder"), ("pose_mlp", "decoder"),
                                                                  ("pose_mlp", "decoder", "tiled"), ("pose_mlp", "partial_slab")}
    assert not _missing(seen, want), f"launch variants that did not occur: {_missing(seen, want)}"


def test_clear_releases_the_last_graph():
    """GenerateEngine.clear() frees the buffers of every cached graph, including the one the body ran last (the engine
    keeps it for its layer helpers): the audits run one signature at a time and rely on it to fit 1320-row graphs."""
    with precision("bf16"):
        model = image_model("dcgan", 64, 1)
        x = frames(3, 2, (1, 64, 64), 4)
        model.p2p_generate_graphed(x, 3, 2)
        eng = model._graphed_engine()
        out = weakref.ref(next(iter(eng._graphs.values())).bufs["out"])
        assert out() is not None
        eng.clear()
        assert out() is None, "a graph buffer outlives GenerateEngine.clear()"
        model.p2p_generate_graphed(x, 3, 2)   # and the engine still captures and replays afterwards
        assert len(eng._graphs) == 1
