"""p2pvg_frame_metrics / p2pvg_pose_metrics (p2pvg_b200/csrc/metrics.cu) and P2PModel.p2p_evaluate against the float64
restatement (tests/metrics_ref.py).

Tolerances: mse rtol 1e-6, psnr 1e-5 dB, ssim 1e-5 absolute; identical frames give mse exactly 0, psnr inf and
|ssim - 1| <= 1e-6.  Poses are scored in fp64 from fp32 inputs: rtol 1e-12."""
import math
import types

import numpy as np
import pytest
import torch

from p2pvg_b200 import metrics
from p2pvg_b200._lib import KernelError, kernels_for
from tests import metrics_ref as R
from tests.test_generate_engine_gpu import draws_for, run

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOL = {"mse": 1e-6, "psnr": 1e-5, "ssim": 1e-5}
CONTENTS = ("uniform", "mnist", "bright", "constant", "identical")


def frame_pair(kind, shape, data_range, g):
    """(pred, gt) fp32 [C, H, W] on the CPU, values in [0, data_range]."""
    if kind == "uniform":
        p, q = torch.rand(shape, generator=g), torch.rand(shape, generator=g)
    elif kind == "mnist":   # mostly near 0 or 1, like rendered digits
        p, q = torch.sigmoid(3 * torch.randn(shape, generator=g)), torch.sigmoid(3 * torch.randn(shape, generator=g))
    elif kind == "bright":  # near-flat and bright: where mean(x^2) - mean(x)^2 cancels most
        p, q = 0.95 + 1e-2 * torch.rand(shape, generator=g), 0.95 + 1e-2 * torch.rand(shape, generator=g)
    elif kind == "constant":
        p, q = torch.full(shape, 0.3), torch.full(shape, 0.7)
    else:
        p = torch.rand(shape, generator=g)
        q = p.clone()
    return (p * data_range).float(), (q * data_range).float()


def check_rows(got, ref, identical=(), what=""):
    """got, ref: float64 [n, 3] (mse, psnr, ssim) as numpy arrays."""
    for r in range(ref.shape[0]):
        (m, p, s), (rm, rp, rs) = got[r], ref[r]
        w = f"{what} row {r}"
        if r in identical:
            assert m == 0.0 and p == math.inf and abs(s - 1) <= 1e-6, f"{w}: {m} {p} {s}"
            continue
        assert abs(m - rm) <= TOL["mse"] * abs(rm), f"{w}: mse {m} vs {rm}"
        assert abs(p - rp) <= TOL["psnr"], f"{w}: psnr {p} vs {rp}"
        assert abs(s - rs) <= TOL["ssim"], f"{w}: ssim {s} vs {rs}"


def as_rows(res):
    return torch.stack([res[k] for k in metrics.FRAME_METRICS], 1).cpu().numpy()


# ---- 1. the kernel against the restatement ------------------------------------------------------------------------------
@pytest.mark.parametrize("data_range", [1.0, 2.0])
@pytest.mark.parametrize("shape", [(1, 7, 8), (1, 12, 36), (1, 64, 64), (3, 64, 64), (3, 128, 128), (4, 128, 128)])
def test_frame_metrics_match_restatement(shape, data_range):
    g = torch.Generator().manual_seed(sum(shape))
    pairs = [frame_pair(k, shape, data_range, g) for k in CONTENTS]
    pred, gt = torch.stack([p for p, _ in pairs]), torch.stack([q for _, q in pairs])
    got = as_rows(metrics.frame_metrics(pred.to(DEV), gt.to(DEV), data_range=data_range))
    ref = R.frame_scores_many(pred.numpy(), gt.numpy(), [(i, i) for i in range(len(CONTENTS))], data_range)
    worst = np.abs(got[:4, 2] - ref[:4, 2]).max()
    print(f"{shape} R={data_range}: worst ssim error {worst:.2e}")
    check_rows(got, ref, identical=(CONTENTS.index("identical"),), what=f"{shape} R={data_range}")


# ---- 2. pair semantics --------------------------------------------------------------------------------------------------
def test_pairs_shared_gt_permuted_and_alone_bit_identical():
    g = torch.Generator().manual_seed(7)
    pred = torch.rand(6, 3, 64, 64, generator=g).to(DEV)
    gt = torch.rand(3, 3, 64, 64, generator=g).to(DEV)
    pairs = torch.tensor([[i, j] for i in range(6) for j in range(3)], dtype=torch.int32)
    perm = torch.randperm(len(pairs), generator=g)
    a = as_rows(metrics.frame_metrics(pred, gt, pairs))
    b = as_rows(metrics.frame_metrics(pred, gt, pairs[perm]))
    again = as_rows(metrics.frame_metrics(pred, gt, pairs))
    assert np.array_equal(a, again), "two launches differ"
    assert np.array_equal(a[perm.numpy()], b), "a pair's result depends on the launch order"
    for r, (i, j) in enumerate(pairs.tolist()):
        alone = as_rows(metrics.frame_metrics(pred, gt, [[i, j]]))
        assert np.array_equal(alone[0], a[r]), f"pair ({i}, {j}) alone differs"
    check_rows(a, R.frame_scores_many(pred.cpu().numpy(), gt.cpu().numpy(), pairs.numpy()))


def test_no_pairs_returns_empty():
    x = torch.rand(2, 1, 8, 8, device=DEV)
    res = metrics.frame_metrics(x, x, torch.zeros(0, 2, dtype=torch.int32))
    assert all(v.shape == (0,) and v.dtype == torch.float64 and v.is_cuda for v in res.values())
    res = metrics.pose_metrics(torch.zeros(2, 17, 3, device=DEV), torch.zeros(2, 17, 3, device=DEV), torch.zeros(0, 2, dtype=torch.int64))
    assert all(v.shape == (0,) for v in res.values())


# ---- 3. a vis_seq-sized launch: dcgan_64, B = 100, 30 frames, 20 samples ---------------------------------------------------
def test_vis_seq_sized_launch():
    T, B, ns, n_past = 30, 100, 20, 1
    frames, pairs = metrics.plan_pairs(T, T, n_past, ns, B)
    assert len(pairs) == 58000
    g = torch.Generator(device=DEV).manual_seed(3)
    pred = torch.rand((T - n_past) * ns * B, 1, 64, 64, device=DEV, generator=g)
    gt = torch.rand(T * B, 1, 64, 64, device=DEV, generator=g)
    a = as_rows(metrics.frame_metrics(pred, gt, pairs))
    b = as_rows(metrics.frame_metrics(pred, gt, pairs))
    assert np.array_equal(a, b)
    pick = np.random.default_rng(0).choice(len(pairs), 500, replace=False)
    sub = pairs[pick].long()
    ref = R.frame_scores_many(pred[sub[:, 0].to(DEV)].cpu().numpy(), gt[sub[:, 1].to(DEV)].cpu().numpy(),
                              [(i, i) for i in range(500)])
    check_rows(a[pick], ref, what="vis_seq")


# ---- 4. rejections ------------------------------------------------------------------------------------------------------
def test_abi_rejects_bad_arguments():
    K = kernels_for(DEV)
    pred = torch.rand(2, 1, 8, 8, device=DEV)
    pairs = torch.zeros(1, 2, dtype=torch.int32, device=DEV)
    out = torch.empty(1, 3, dtype=torch.float64, device=DEV)
    ok = dict(pred=pred, gt=pred, pairs=pairs, n_pairs=1, C=1, H=8, W=8, data_range=1.0, out=out)
    K.frame_metrics(**ok)
    torch.cuda.synchronize()
    odd = torch.empty(64, device=DEV)[1:]   # 4 bytes past a 16-byte boundary
    bad = [dict(pred=None), dict(gt=None), dict(pairs=None), dict(out=None), dict(pred=odd), dict(gt=odd), dict(out=odd),
           dict(pairs=torch.empty(8, dtype=torch.uint8, device=DEV)[1:]), dict(C=0), dict(H=6), dict(W=4), dict(W=10),
           dict(n_pairs=-1), dict(data_range=0.0), dict(data_range=-1.0), dict(data_range=math.inf), dict(data_range=math.nan),
           dict(W=132), dict(C=1 << 16, H=256, W=128)]
    for b in bad:
        with pytest.raises(KernelError):
            K.frame_metrics(**{**ok, **b})
    pose = torch.zeros(2, 17, 3, device=DEV)
    pout = torch.empty(1, 2, dtype=torch.float64, device=DEV)
    okp = dict(pred=pose, gt=pose, pairs=pairs, n_pairs=1, J=17, out=pout)
    K.pose_metrics(**okp)
    for b in (dict(pred=None), dict(gt=None), dict(pairs=None), dict(out=None), dict(out=odd), dict(J=0), dict(n_pairs=-1)):
        with pytest.raises(KernelError):
            K.pose_metrics(**{**okp, **b})
    K.frame_metrics(**{**ok, "n_pairs": 0})
    K.frame_metrics(**{**ok, "n_pairs": 0, "pairs": None, "out": None})   # zero pairs: pairs and out are never read
    K.pose_metrics(**{**okp, "n_pairs": 0, "pairs": None, "out": None})
    torch.cuda.synchronize()


def test_wrapper_rejects_before_launch():
    x = torch.rand(3, 1, 8, 8, device=DEV)
    K = kernels_for(DEV)
    n0 = K.launches
    cases = [dict(pairs=[[3, 0]]), dict(pairs=[[0, -1]]), dict(pairs=[[0, 3]]), dict(pairs=torch.zeros(2, 3, dtype=torch.int32)),
             dict(pairs=torch.zeros(1, 2)), dict(pred=x.double()), dict(gt=x.half()), dict(pred=x.transpose(2, 3)),
             dict(pred=x.cpu()), dict(gt=x.cpu()), dict(gt=torch.rand(3, 1, 8, 12, device=DEV)), dict(data_range=0.0),
             dict(data_range=math.nan), dict(pred=torch.rand(3, 1, 8, 10, device=DEV)), dict(pred=x[0])]
    for c in cases:
        kw = dict(pred=x, gt=x, pairs=None, data_range=1.0)
        kw.update(c)
        with pytest.raises(ValueError):
            metrics.frame_metrics(kw["pred"], kw["gt"], kw["pairs"], kw["data_range"])
    with pytest.raises(ValueError):
        metrics.frame_metrics(x, x[:2])   # pairs=None needs as many gt frames as pred frames
    p = torch.zeros(2, 17, 3, device=DEV)
    for a, b, pr in ((p, p, [[2, 0]]), (p.cpu(), p, None), (p.double(), p, None), (p, torch.zeros(2, 17, 2, device=DEV), None)):
        with pytest.raises(ValueError):
            metrics.pose_metrics(a, b, pr)
    assert K.launches == n0


# ---- 5. the pose kernel -------------------------------------------------------------------------------------------------
def test_pose_metrics_match_restatement():
    g = torch.Generator().manual_seed(5)
    pred, gt = torch.randn(40, 17, 3, generator=g), torch.randn(12, 17, 3, generator=g)
    pred[:12] = gt   # identical poses
    pairs = torch.cat([torch.stack([torch.arange(12), torch.arange(12)], 1),
                       torch.stack([torch.randint(0, 40, (50,), generator=g), torch.randint(0, 12, (50,), generator=g)], 1)])
    res = metrics.pose_metrics(pred.to(DEV), gt.to(DEV), pairs)
    got = torch.stack([res["mse"], res["mpjpe"]], 1).cpu().numpy()
    ref = R.pose_scores_many(pred.numpy(), gt.numpy(), pairs.numpy())
    assert (got[:12] == 0).all()
    np.testing.assert_allclose(got, ref, rtol=1e-12, atol=0)


# ---- 6. P2PModel.p2p_evaluate end to end --------------------------------------------------------------------------------
def make_model(backbone, C, B, n_past, seed=0):
    from p2pvg_b200.models import dcgan_64, dcgan_128, h36m_mlp, vgg_64, vgg_128
    from p2pvg_b200.models.p2p_model import P2PModel
    net = dict(dcgan_64=dcgan_64, dcgan_128=dcgan_128, vgg_64=vgg_64, vgg_128=vgg_128, h36m_mlp=h36m_mlp)[backbone]
    opt = types.SimpleNamespace(dataset="h36m" if backbone == "h36m_mlp" else "mnist", backbone_net=net, lr=1e-3, beta1=0.9,
                                beta=1e-4, weight_cpc=100.0, weight_align=0.5, skip_prob=0.5, n_past=n_past, last_frame_skip=False,
                                batch_size=B)
    torch.manual_seed(seed)
    model = P2PModel(B, C, 128, 10, 256, 1, 1, 2, opt=opt)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():   # move every parameter off the tiny reference initialisation so samples differ visibly
        for p in model.parameters():
            p.add_(0.05 * torch.randn(p.shape, generator=g))
    return model.cuda().eval()


def restated(seq, x, frames, gts, ns, pose, data_range):
    """float64 [metric][nsample, F, B] scores of the stacked generated frames."""
    names = metrics.POSE_METRICS if pose else metrics.FRAME_METRICS
    B = x.shape[1]
    out = np.zeros((len(names), ns, len(frames), B))
    for s in range(ns):
        for fi, (i, t) in enumerate(zip(frames, gts)):
            for b in range(B):
                p, q = seq[s][i][b].double().cpu().numpy(), x[t][b].double().cpu().numpy()
                out[:, s, fi, b] = R.pose_scores(p, q) if pose else R.frame_scores(p, q, data_range)
    return dict(zip(names, out))


def check_evaluate(model, x, ns, mode, L=None, data_range=1.0, np_seed=4):
    pose = model.is_pose
    T, B = x.shape[0], x.shape[1]
    L = T if L is None else L
    n_past = model.opt.n_past
    draws = draws_for(L - 1, ns * B, model.z_dim, seed=L + ns)
    ev = run(lambda: model.p2p_evaluate(x, nsample=ns, len_output=None if L == T else L, model_mode=mode, data_range=data_range),
             np_seed, draws)
    hid_ev = {m: [(h.clone(), c.clone()) for h, c in getattr(model, m).hidden] for m in ("posterior", "prior", "frame_predictor")}
    seq = run(lambda: model.p2p_generate_graphed(x, L, L - 1, model_mode=mode, nsample=ns), np_seed, draws)
    seq = [seq] if ns == 1 else seq
    for m, hc in hid_ev.items():
        for (h1, c1), (h2, c2) in zip(hc, getattr(model, m).hidden):
            assert torch.equal(h1, h2) and torch.equal(c1, c2), f".hidden of {m} differs from p2p_generate_graphed's"
    frames = list(range(n_past, L)) if L == T else [L - 1]
    gts = frames if L == T else [T - 1]
    assert ev["frames"] == frames
    ref = restated(seq, x, frames, gts, ns, pose, data_range)
    for k, r in ref.items():
        got = ev[k]
        assert got.shape == (ns, len(frames), B) and got.dtype == torch.float64 and got.is_cuda, k
        got = got.cpu().numpy()
        if k == "mse":
            assert np.all(np.abs(got - r) <= (1e-12 if pose else TOL["mse"]) * np.abs(r)), f"{k}: {np.abs(got - r).max()}"
        elif k == "mpjpe":
            np.testing.assert_allclose(got, r, rtol=1e-12, atol=0)
        else:
            assert np.abs(got - r).max() <= TOL[k], f"{k}: {np.abs(got - r).max()}"
        idx, curve = ev["best"][k]
        assert idx.shape == (B,) and curve.shape == (len(frames), B)
        assert torch.equal(curve, ev[k][idx, :, torch.arange(B, device=idx.device)].T), k
        mean = r.mean(1)   # [ns, B]
        hi = metrics.HIGHER_IS_BETTER[k]
        want = mean.argmax(0) if hi else mean.argmin(0)
        tol = TOL.get(k, 1e-12) * (np.abs(mean).max() if k in ("mse", "mpjpe") else 1)
        if ns == 1:
            assert (idx == 0).all(), k
        for b in range(B if ns > 1 else 0):
            srt = np.sort(mean[:, b])
            gap = (srt[-1] - srt[-2]) if hi else (srt[1] - srt[0])
            if gap > tol:
                assert idx[b].item() == want[b], f"{k} best sample of row {b}"
    return ev


@pytest.mark.parametrize("n_past,mode", [(1, "full"), (2, "full"), (1, "prior"), (2, "prior")])
def test_evaluate_dcgan64(n_past, mode):
    T, B = 6, 3
    model = make_model("dcgan_64", 1, B, n_past)
    x = torch.rand(T, B, 1, 64, 64, generator=torch.Generator().manual_seed(n_past)).cuda()
    check_evaluate(model, x, ns=4, mode=mode)
    check_evaluate(model, x, ns=1, mode=mode)


@pytest.mark.parametrize("L", [4, 8])
def test_evaluate_dcgan64_control_point_only(L):
    T, B = 6, 2
    model = make_model("dcgan_64", 1, B, 1)
    x = torch.rand(T, B, 1, 64, 64, generator=torch.Generator().manual_seed(L)).cuda()
    ev = check_evaluate(model, x, ns=3, mode="full", L=L)
    assert ev["frames"] == [L - 1] and ev["ssim"].shape == (3, 1, B)


@pytest.mark.parametrize("backbone,C,W", [("dcgan_128", 3, 128), ("vgg_64", 3, 64), ("vgg_128", 3, 128)])
def test_evaluate_rgb_backbones(backbone, C, W):
    T, B = 5, 2
    model = make_model(backbone, C, B, 2)
    x = torch.rand(T, B, C, W, W, generator=torch.Generator().manual_seed(W)).cuda()
    check_evaluate(model, x, ns=3, mode="full", data_range=1.0)


def test_evaluate_h36m_mlp():
    T, B = 8, 4
    model = make_model("h36m_mlp", 1, B, 2)
    x = torch.randn(T, B, 17, 3, generator=torch.Generator().manual_seed(2)).cuda()
    ev = check_evaluate(model, x, ns=5, mode="full")
    assert set(ev) == {"frames", "mse", "mpjpe", "best"}
    ev = run(lambda: model.p2p_evaluate((x[..., :2].contiguous(), x, torch.zeros(B, dtype=torch.int64)), nsample=2),
             1, draws_for(T - 1, 2 * B, model.z_dim, 1))
    assert ev["mse"].shape == (2, T - 2, B)


def test_evaluate_one_launch_on_a_cached_signature():
    from p2pvg_b200 import infer
    T, B, ns = 6, 2, 3
    model = make_model("dcgan_64", 1, B, 1)
    x = torch.rand(T, B, 1, 64, 64, generator=torch.Generator().manual_seed(9)).cuda()
    draws = draws_for(T - 1, ns * B, model.z_dim, 1)
    first = run(lambda: model.p2p_evaluate(x, nsample=ns), 1, draws)
    base, view = kernels_for(x.device), infer.kernels_for(x.device)
    n_graphs, n_base, n_view = len(model._gen_engine._graphs), base.launches, view.launches
    again = run(lambda: model.p2p_evaluate(x, nsample=ns), 1, draws)
    torch.cuda.synchronize()
    assert base.launches - n_base == 1 and view.launches == n_view
    assert len(model._gen_engine._graphs) == n_graphs
    for k in metrics.FRAME_METRICS:
        assert torch.equal(first[k], again[k]), k
    # the graph is shared with p2p_generate_graphed of the same arguments
    run(lambda: model.p2p_generate_graphed(x, T, T - 1, nsample=ns), 1, draws)
    assert len(model._gen_engine._graphs) == n_graphs


def test_evaluate_rejections():
    T, B = 4, 1
    model = make_model("dcgan_64", 1, B, 2)
    x = torch.rand(T, B, 1, 64, 64).cuda()
    for kw in (dict(len_output=2), dict(len_output=1), dict(data_range=0.0), dict(data_range=-1.0)):
        with pytest.raises(ValueError):
            model.p2p_evaluate(x, **kw)
    model.train()
    with pytest.raises(ValueError):
        model.p2p_evaluate(x)
