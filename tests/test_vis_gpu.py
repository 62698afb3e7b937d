"""p2pvg_b200.visualize on the GPU: the p2pvg_vis_canvas kernel and vis_seq against the reference's own pictures
(tests/golden/vis_seq.pt: the kernel bit for bit on the composition cases, whose samples the fixture redraws; vis_seq with the
reference's draws on the generation cases, against a 2048-value digest of each canvas) and against the restated reference
vis_seq over the eager p2p_generate (tests/vis_ref.py).

Tolerances on the canvases: those of generation (fp32 2e-4 worst / 2e-5 mean, bf16 4e-2 / 6e-3 on frames in [0, 1]); pose
pictures are images the stub visualizer quantises to 1/255, so there a pixel may move by one step."""
import hashlib
import os
import sys
import types

import numpy as np
import pytest
import torch

from oracle import p2p_oracle as O
from p2pvg_b200 import visualize as V
from p2pvg_b200._lib import KernelError, kernels_for
from tests.test_generate_engine_gpu import TOL, precision
from tests.test_pose_generate_gpu import pose_model, pose_opt
from tests.vis_ref import FrameSource, PoseStub, Recorder, case_input, compose_ref, vis_seq_ref

pytestmark = pytest.mark.gpu
FIX = os.path.join(os.path.dirname(__file__), "golden", "vis_seq.pt")
STEP = 1 / 255 + 1e-6


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.fixture(scope="module")
def fix():
    return torch.load(FIX, weights_only=False)


@pytest.fixture
def rec(monkeypatch):
    r = Recorder()
    monkeypatch.setitem(sys.modules, "imageio", r.imageio)
    tv = types.ModuleType("torchvision")
    tv.utils = r.vutils
    monkeypatch.setitem(sys.modules, "torchvision", tv)
    monkeypatch.setitem(sys.modules, "torchvision.utils", r.vutils)
    return r


def fixture_model(c):
    o = dict(c["opt"])
    if c["spec"]["net"] == "mlp":
        model = pose_model(O.build_state(c["cfg"], seed=c["init_seed"]), pose_opt(o["batch_size"], o["n_past"],
                                                                                   o["last_frame_skip"], o["skip_prob"]), c["cfg"])
    else:
        from tests.test_generate_gpu import build_model
        model = build_model(c)
    model.opt.nsample, model.opt.log_dir = c["nsample"], "LOGDIR"
    return model


def fixture_stores(c, dev):
    """The ground truth and the FrameSource samples of a composition case, as vis_seq's two stores."""
    ns, L, nb, T, C = c["nsample"], c["spec"]["L"], c["n_block"], c["spec"]["T"], c["spec"]["channels"]
    x = case_input(c["spec"])
    s0 = x[:, :nb].reshape(T * nb, C, 64, 64).contiguous().to(dev)
    smp = FrameSource(c["spec"]["src_seed"], c["spec"]["zero"]).samples(x, ns, L)
    s1 = smp[:, :, :nb].reshape(ns * L * nb, C, 64, 64).contiguous().to(dev)
    return s0, s1, C


def plan(c, gt_ref, sample_ref):
    np.random.seed(c["np_seed"])
    for _ in range(c["nsample"]):
        np.random.uniform(0, 1, c["spec"]["L"] - 1)
    return V.plan_tiles(c["spec"]["T"], c["spec"]["L"], c["n_block"], c["nsample"], gt_ref, sample_ref)


# (a) ---------------------------------------------------------------------------------------------------------------------
def test_kernel_bit_identical_to_reference(fix):
    cases = [c for c in fix["cases"] if c["spec"]["net"] == "source"]
    assert len(cases) == 3
    for c in cases:
        ns, L, nb = c["nsample"], c["spec"]["L"], c["n_block"]
        s0, s1, C = fixture_stores(c, "cuda")
        tiles = plan(c, lambda t: (0, t * nb), lambda s, t: (1, (s * L + t) * nb))
        canvas, video, gif = V.compose(s0, s1, tiles, C, 64)
        torch.cuda.synchronize()
        assert sha(canvas.cpu().numpy()) == c["canvas"]["sha"], c["case"]
        assert sha(video.unsqueeze(0).cpu().numpy()) == c["video"]["sha"], c["case"]
        assert sha(gif.cpu().numpy()) == c["gif"]["sha"], c["case"]


# (b) ---------------------------------------------------------------------------------------------------------------------
def inject_eps(monkeypatch, eps):
    """vis_seq's torch.randn draws replaced by the reference's, in call order."""
    pos = [0]

    def draws(B, z, dev, n_exec, nb):
        k = pos[0]
        pos[0] += 2 * n_exec
        return eps[k:k + 2 * n_exec].view(n_exec, 2, B, z)[:, :, :nb].to(dev)
    monkeypatch.setattr(V, "_eps", draws)
    return pos


@pytest.mark.parametrize("case", ["d64_c1_eq", "d64_c1_above", "d64_c3_below", "h36m"])
def test_vis_seq_fp32_against_reference(fix, rec, monkeypatch, case):
    c = next(c for c in fix["cases"] if c["case"] == case)
    sp = c["spec"]
    with precision("fp32"):
        model = fixture_model(c)
        x = case_input(sp)
        x = tuple(t.cuda() for t in x) if sp["net"] == "mlp" else x.cuda()
        pos = inject_eps(monkeypatch, c["eps"])
        stub = PoseStub() if sp["net"] == "mlp" else None
        np.random.seed(c["np_seed"])
        V.vis_seq(model, x, 7, sp["L"], model_mode=sp["mode"], recon_mode=sp["recon"], skip_frame=sp["skip"],
                  h36m_visualizer=stub, writer=rec, opt=model.opt)
    assert pos[0] == c["n_calls"]
    st, ref = np.random.get_state(), c["np_state_after"]
    assert st[0] == ref[0] and np.array_equal(st[1], ref[1]) and st[2:] == ref[2:]
    (png, canvas), = rec.saved
    (gifn, gif), = rec.gifs
    (it, img, istep), = rec.images
    (vt, vid, vstep, fps), = rec.videos
    assert (png, gifn) == c["names"] and (it, vt) == c["tags"] and (istep, vstep) == c["steps"] and fps == c["fps"] == 2
    assert img.dtype == np.float32 and vid.dtype == np.float32 and all(g.dtype == np.uint8 for g in gif)
    assert tuple(canvas.shape) == c["canvas"]["shape"] and vid.shape == c["video"]["shape"]
    assert len(gif) == c["gif"]["n"] and (len(gif), *gif[0].shape) == c["gif"]["shape"]
    ns, L, nb, T = c["nsample"], sp["L"], c["n_block"], sp["T"]
    if sp["net"] == "mlp":
        assert len(stub.calls) == len(c["set_data"])
        for (p, v), (q, w) in zip(stub.calls, c["set_data"]):
            assert v == w and p.shape == q.shape and np.abs(p - q).max() <= 3e-4
        imgs = [stub.set_data(p, v) for p, v in c["set_data"]]
        a = lambda ims: torch.from_numpy((np.stack(ims, 1).astype(np.float64) / 255.).astype(np.float32)).permute(0, 1, 4, 2, 3)  # noqa: E731
        smp = torch.stack([a(imgs[s * nb:(s + 1) * nb]) for s in range(ns)])
        want = compose_ref(a(imgs[ns * nb:])[:T], smp, T, L, c["s_lists"])[0]
        e = (canvas - want).abs()
        assert e.max().item() <= STEP and e.mean().item() <= 1e-3
    else:
        # the reference canvas's digest: 2048 values at fixed positions, its sum and its largest magnitude
        d = c["canvas"]["digest"]
        got = canvas.double().reshape(-1)
        tmax, tmean = TOL["fp32"]
        e = (got[d["idx"]] - d["samples"]).abs()
        assert e.max().item() <= tmax and e.mean().item() <= tmean, (e.max().item(), e.mean().item())
        assert abs(got.sum().item() - d["sum"]) <= tmean * got.numel() and abs(got.abs().max().item() - d["absmax"]) <= tmax
    assert np.array_equal(img, canvas.numpy())


# (c) ---------------------------------------------------------------------------------------------------------------------
def bench_model(kind, B, ns):
    from p2pvg_b200.models import dcgan_64, h36m_mlp, vgg_64
    from p2pvg_b200.models.p2p_model import P2PModel
    pose = kind == "pose"
    net = {"dcgan64": dcgan_64, "vgg64": vgg_64, "pose": h36m_mlp}[kind]
    opt = types.SimpleNamespace(dataset="h36m" if pose else "mnist", backbone_net=net, lr=1e-3, beta1=0.9, beta=1e-4,
                                weight_cpc=100.0, weight_align=0.5, skip_prob=0.5, n_past=1, last_frame_skip=False, batch_size=B,
                                nsample=ns, log_dir="LOG")
    torch.manual_seed(1)
    C = 3 if kind == "vgg64" else 1
    return P2PModel(B, C, 128, 10, 512 if pose else 256, 1, 1, 2, opt=opt).cuda().eval(), C


def bench_input(kind, T, B, C):
    g = torch.Generator().manual_seed(5)
    if kind == "pose":
        return (torch.randn(T, B, 17, 2, generator=g).cuda(), 3 * torch.randn(T, B, 17, 3, generator=g).cuda(),
                torch.arange(B).cuda() % 4)
    return torch.rand(T, B, C, 64, 64, generator=g).cuda()


@pytest.mark.parametrize("kind,B,T,L,skip_frame", [("dcgan64", 100, 30, 30, False), ("vgg64", 128, 30, 30, False),
                                                    ("dcgan64", 100, 10, 12, True), ("pose", 10, 10, 12, False),
                                                    ("pose", 10, 10, 8, True)])
def test_vis_seq_bf16_against_eager(rec, kind, B, T, L, skip_frame):
    """The central claim: the drop-in's vis_seq shows the reference's pictures (eager p2p_generate on the whole batch, within
    generation tolerance) and leaves NumPy's and torch's CUDA random streams exactly where the eager calls leave them."""
    ns = 20
    model, C = bench_model(kind, B, ns)
    x = bench_input(kind, T, B, C)
    outs, states = [], []
    for fn in (vis_seq_ref, V.vis_seq):
        np.random.seed(11)
        torch.cuda.manual_seed(12)
        kw = dict(rec=rec) if fn is vis_seq_ref else {}
        stub = PoseStub() if kind == "pose" else None
        outs.append(fn(model, x, 3, L, model_mode="full", recon_mode="test", skip_frame=skip_frame, h36m_visualizer=stub,
                       writer=rec, opt=model.opt, **kw))
        torch.cuda.synchronize()
        states.append((np.random.get_state(), torch.cuda.get_rng_state(), stub.calls if stub else None))
    (a, b) = states
    assert a[0][0] == b[0][0] and np.array_equal(a[0][1], b[0][1]) and a[0][2:] == b[0][2:]
    assert torch.equal(a[1], b[1])
    if kind == "pose":
        assert len(a[2]) == len(b[2]) and all(v == w and np.abs(p - q).max() <= 3e-4 for (p, v), (q, w) in zip(a[2], b[2]))
    for k, (r, g) in enumerate(zip(outs[0][:2], outs[1][:2])):
        e = (r.float().cpu() - g.float().cpu()).abs()
        tmax, tmean = (STEP, 1e-3) if kind == "pose" else TOL["bf16"]
        assert e.max().item() <= tmax and e.mean().item() <= tmean, (k, e.max().item(), e.mean().item())
    ga, gb = outs[0][2], outs[1][2].cpu().numpy()
    assert ga.shape == gb.shape and ga.dtype == gb.dtype == np.uint8
    assert [s[0] for s in rec.saved[:1]] == [s[0] for s in rec.saved[1:]] and rec.images[0][0] == rec.images[1][0]


# (d) ---------------------------------------------------------------------------------------------------------------------
def test_rejections_before_any_draw(rec):
    model, C = bench_model("dcgan64", 4, 3)
    x = bench_input("dcgan64", 6, 4, C)
    bad = []
    m2, _ = bench_model("dcgan64", 4, 1)
    bad.append((m2, x, 6))                                   # nsample < 2
    m3, _ = bench_model("dcgan64", 12, 3)
    bad.append((m3, bench_input("dcgan64", 6, 4, C), 6))     # fewer rows than n_block
    m4, _ = bench_model("dcgan64", 4, 3)
    m4.train()
    bad.append((m4, x, 6))                                   # training mode
    m5, _ = bench_model("dcgan64", 4, 3)
    m5.cpu()
    bad.append((m5, x, 6))                                   # CPU model
    bad.append((model, x, 1))                                # output_len < 2
    bad.append((model, x[:, :, :, :32, :32].contiguous(), 6))  # frame shape the backbone does not take
    for m, xx, L in bad:
        np.random.seed(3)
        torch.cuda.manual_seed(4)
        st, cst = np.random.get_state(), torch.cuda.get_rng_state()
        n = kernels_for(torch.device("cuda")).launches
        with pytest.raises(ValueError):
            V.check_vis_seq(m, xx, L, "full", False, m.opt)
        with pytest.raises(ValueError):
            V.vis_seq(m, xx, 0, L, skip_frame=False, writer=rec, opt=m.opt)
        assert np.array_equal(np.random.get_state()[1], st[1]) and np.random.get_state()[2] == st[2]
        assert torch.equal(torch.cuda.get_rng_state(), cst)
        assert kernels_for(torch.device("cuda")).launches == n
    assert not rec.saved and not rec.gifs


# (e) ---------------------------------------------------------------------------------------------------------------------
def test_kernel_rejects_malformed_arguments():
    K = kernels_for(torch.device("cuda"))
    s = torch.zeros(4, 1, 8, 8, device="cuda")
    r_len, nb, H = 2, 1, 8
    canvas = torch.empty(3, nb * 6 * H, r_len * H, device="cuda")
    video = torch.empty(r_len, 3, nb * H, 6 * H, device="cuda")
    gif = torch.empty(r_len, nb * H, 6 * H, 3, device="cuda", dtype=torch.uint8)
    good = np.zeros((r_len, nb, 6, 3), np.int32)
    tdev = torch.empty(good.size, device="cuda", dtype=torch.int32)
    K.vis_canvas(s, 4, None, 0, 1, H, good, tdev, r_len, nb, canvas, video, gif)
    for C, Hh, tweak in ((2, H, None), (4, H, None), (1, 0, None), (1, 129, None), (1, H, (0, 1, 4)), (1, H, (1, 0, 0)),
                         (1, H, (0, -2, 0)), (1, H, (2, 0, 0)), (1, H, (0, 0, 3)), (1, H, (0, 0, -1))):
        t = good.copy()
        if tweak is not None:
            t[1, 0, 3] = tweak
        with pytest.raises(KernelError):
            K.vis_canvas(s, 4, None, 0, C, Hh, t, tdev, r_len, nb, canvas, video, gif)
    with pytest.raises(ValueError):
        V.compose(s.double(), None, good, 1, H)
