"""p2pvg_moving_mnist / p2pvg_b200.data.MovingMNIST: Moving MNIST batches rendered on the device.

The fixtures tests/golden/mmnist_*.pt were written by the unmodified reference renderer (make_golden_mnist.py) from seeded
draws; the kernel fed the same draws and digits must reproduce every sequence bit for bit."""
import ctypes
import hashlib
import os
import sys
import types

import numpy as np
import pytest
import torch
from scipy import stats

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
CASES = [(det, nd, S) for det in (False, True) for nd in (1, 2, 3) for S in (64, 128)]   # as make_golden_mnist.py writes them


def case_name(det, nd, S):
    return f"mmnist_det{int(det)}_nd{nd}_s{S}.pt"


def kernels():
    from p2pvg_b200._lib import kernels_for
    return kernels_for("cuda")


def sha(x):
    return hashlib.sha256(x.contiguous().cpu().numpy().tobytes()).hexdigest()


@pytest.mark.parametrize("det,nd,S", CASES, ids=[case_name(*c)[:-3] for c in CASES])
def test_fixture_sequences_bit_identical(det, nd, S):
    digits = torch.load(os.path.join(GOLDEN, "mmnist_digits.pt"))["digits"].cuda()
    rec = torch.load(os.path.join(GOLDEN, case_name(det, nd, S)))
    draws = rec["draws"].cuda()
    B = len(draws)
    for T, key in ((rec["max_seq_len"], "sha256_full"), (rec["t_short"], "sha256_short")):
        out = torch.full((T, B, 1, S, S), float("nan"), device="cuda")
        kernels().moving_mnist(digits, draws, out, T, B, S, nd, det)
        bad = [b for b in range(B) if sha(out[:, b]) != rec[key][b]]
        detail = ""
        if bad and "frames" in rec and 0 in bad:
            n = min(T, len(rec["frames"]))
            detail = f"; sequence 0 max |diff| {(out[:n, 0].cpu() - rec['frames'][:n]).abs().max().item()}"
        assert not bad, f"T={T}: sequences {bad} differ from the reference{detail}"


def square_digit():
    return torch.full((1, 32, 32), 255, dtype=torch.uint8)


def positions(frames):
    """(y, x) of the top-left corner of the single 32x32 square of ones in each [.., S, S] frame."""
    m = frames > 0
    y = m.any(-1).float().argmax(-1)
    x = m.any(-2).float().argmax(-1)
    return y, x


def test_device_draws_positions_values_and_seed():
    from p2pvg_b200.data import MovingMNIST
    S, T, B = 64, 12, 64
    np.random.seed(3)
    sq = next(MovingMNIST(square_digit(), B, T, 0, image_size=S, num_digits=1,
                          generator=torch.Generator("cuda").manual_seed(1)))
    assert tuple(sq.shape) == (T, B, 1, S, S) and sq.dtype == torch.float32 and sq.is_cuda
    y, x = positions(sq[:, :, 0])
    assert int(y.min()) >= 0 and int(x.min()) >= 0 and int(y.max()) <= S - 33 and int(x.max()) <= S - 33
    # every frame is exactly one whole digit: the square never leaves the frame
    assert torch.equal(sq.sum((2, 3, 4)), torch.full((T, B), 1024.0, device="cuda"))

    digits = torch.randint(0, 256, (10, 32, 32), dtype=torch.uint8, generator=torch.Generator().manual_seed(0))
    batches = []
    for _ in range(2):
        np.random.seed(4)
        mm = MovingMNIST(digits, 32, 20, 3, image_size=128, num_digits=3, generator=torch.Generator("cuda").manual_seed(9))
        batches.append([next(mm) for _ in range(3)])
    for a, b in zip(*batches):
        assert torch.equal(a, b)
        assert float(a.min()) >= 0.0 and float(a.max()) <= 1.0
    assert not torch.equal(batches[0][0][:14], batches[0][1][:14])


def test_first_frame_position_and_velocity_are_uniform():
    from p2pvg_b200.data import MovingMNIST
    S, B = 64, 8192
    np.random.seed(0)
    x = next(MovingMNIST(square_digit(), B, 2, 0, image_size=S, num_digits=1, generator=torch.Generator("cuda").manual_seed(5)))
    y, xx = positions(x[:, :, 0])
    sy0, sx0 = y[0].cpu().numpy(), xx[0].cpu().numpy()
    for v in (sx0, sy0):
        assert stats.chisquare(np.bincount(v, minlength=S - 32)).pvalue > 1e-3
    # a step that bounces off no wall moves by exactly (dx, dy)
    inner = (sx0 >= 4) & (sx0 <= S - 37) & (sy0 >= 4) & (sy0 <= S - 37)
    dx = xx[1].cpu().numpy()[inner] - sx0[inner]
    dy = y[1].cpu().numpy()[inner] - sy0[inner]
    assert inner.sum() > 3000
    for d in (dx, dy):
        assert d.min() >= -4 and d.max() <= 4
        assert stats.chisquare(np.bincount(d + 4, minlength=9)).pvalue > 1e-3


def test_sequence_lengths_follow_numpy_global_stream():
    from p2pvg_b200.data import MovingMNIST
    mm = MovingMNIST(square_digit(), 2, 30, 5, generator=torch.Generator("cuda").manual_seed(0))
    np.random.seed(11)
    got = [len(next(mm)) for _ in range(25)]
    np.random.seed(11)
    want = [np.random.randint(30 - 10, 30 + 1) for _ in range(25)]
    assert got == want and len(set(got)) > 3


def c2_model(B):
    from p2pvg_b200.models import dcgan_64
    from p2pvg_b200.models.p2p_model import P2PModel
    opt = types.SimpleNamespace(dataset="mnist", backbone_net=dcgan_64, lr=1e-3, beta1=0.9, beta=1e-4, weight_cpc=100.0,
                                weight_align=0.5, skip_prob=0.0, n_past=1, last_frame_skip=False, batch_size=B)
    torch.manual_seed(1)
    return P2PModel(B, 1, 128, 10, 256, 1, 1, 2, opt=opt).cuda()


def test_c2_steps_from_rendered_batches_equal_host_frames(monkeypatch):
    from p2pvg_b200.data import MovingMNIST
    monkeypatch.setenv("P2PVG_GRAPH", "0")
    monkeypatch.setenv("P2PVG_PRECISION", "bf16")
    B = 256
    digits = torch.randint(0, 256, (50, 32, 32), dtype=torch.uint8, generator=torch.Generator().manual_seed(1))
    runs, frames = [], []
    for fed in ("device", "host"):
        model = c2_model(B)
        model.train()
        mm = MovingMNIST(digits, B, 30, 2, generator=torch.Generator("cuda").manual_seed(2))
        np.random.seed(0)
        losses = []
        for i in range(2):
            if fed == "device":
                x = next(mm)
                frames.append(x.cpu())
            else:
                np.random.randint(30 - 4, 30 + 1)   # the draw MovingMNIST makes, so that forward sees the same NumPy stream
                x = frames[i].pin_memory().cuda(non_blocking=True)
            torch.manual_seed(100 + i)
            losses.append(np.array(model(x, 0, len(x) - 1), dtype=np.float64))
        runs.append(losses)
        del model
        torch.cuda.empty_cache()
    for a, b in zip(*runs):
        assert np.all(np.isfinite(a))
        np.testing.assert_allclose(a, b, rtol=1e-5, atol=0)


def test_dropin_mnist_generator_reads_idx_files(tmp_path, monkeypatch):
    import gzip
    from p2pvg_b200.data import load_mnist_digits
    raw = tmp_path / "MNIST" / "raw"
    raw.mkdir(parents=True)
    rs = np.random.RandomState(0)
    for name, n in (("train", 9), ("t10k", 5)):
        imgs = rs.randint(0, 256, (n, 28, 28)).astype(np.uint8)
        hdr = b"".join(v.to_bytes(4, "big") for v in (0x803, n, 28, 28))
        with gzip.open(raw / f"{name}-images-idx3-ubyte.gz", "wb") as f:
            f.write(hdr + imgs.tobytes())
    monkeypatch.setenv("P2PVG_REF", "")
    monkeypatch.syspath_prepend(os.path.join(ROOT, "dropin"))
    for m in ("data", "data.data_utils"):
        monkeypatch.delitem(sys.modules, m, raising=False)
    import data.data_utils as du
    try:
        opt = types.SimpleNamespace(dataset="mnist", data_root=str(tmp_path), max_seq_len=12, delta_len=3, image_width=64,
                                    num_digits=2, batch_size=4)
        train, test = du.load_dataset(opt)
        assert len(train) == 9 and len(test) == 5 and train.max_seq_len == 12
        assert torch.equal(train.digits, load_mnist_digits(str(tmp_path), train=True))
        for ds, is_train in ((train, True), (test, False)):
            gen = du.get_data_generator(ds, train=is_train, opt=opt)
            for _ in range(3):
                x = next(gen)
                assert x.is_cuda and x.dtype == torch.float32 and 6 <= len(x) <= 12
                assert tuple(x.shape[1:]) == (4, 1, 64, 64) and float(x.max()) > 0 and float(x.max()) <= 1
    finally:
        for m in ("data", "data.data_utils"):
            sys.modules.pop(m, None)


def test_kernel_rejects_bad_arguments():
    from p2pvg_b200._lib import load_library
    lib = load_library()
    T, B, S, nd = 3, 2, 64, 2
    digits = torch.zeros(4, 32, 32, dtype=torch.uint8, device="cuda")
    draws = torch.zeros(B, nd, 5 + 4 * T, dtype=torch.int32, device="cuda")
    out = torch.empty(T, B, 1, S, S, device="cuda")
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    P = ctypes.c_void_p

    def call(dig=digits.data_ptr(), n_digits=4, dr=draws.data_ptr(), stride=5 + 4 * T, o=out.data_ptr(), S=S, nd=nd):
        return lib.p2pvg_moving_mnist(P(dig), n_digits, P(dr), stride, P(o), T, B, S, nd, 0, stream)

    assert call() == 0
    torch.cuda.synchronize()
    for kw in (dict(S=32), dict(S=30), dict(S=66), dict(nd=0), dict(nd=5), dict(stride=5 + 4 * T - 1), dict(dig=None),
               dict(dr=None), dict(o=None), dict(n_digits=0)):
        assert call(**kw) == -1, kw
