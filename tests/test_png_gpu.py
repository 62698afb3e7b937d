"""p2pvg_png_encode on the GPU: every file decodes, with PIL and with the NumPy reader of tests/png_ref.py, to exactly the
pixels of the file torchvision.utils.save_image (or TensorBoard's image summary) writes for the same tensor."""
import io
import os
import sys

import numpy as np
import pytest
import torch
import torchvision.utils as vutils
from PIL import Image

from p2pvg_b200 import png
from tests.png_ref import mnist_canvas, read_png, rgb_canvas

pytestmark = pytest.mark.gpu


def pil_pixels(data):
    return np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))


def torchvision_file(t):
    buf = io.BytesIO()
    vutils.save_image(t.cpu(), buf, format="png")
    return buf.getvalue()


def check_file(data, t):
    """data decodes with both readers to the pixels of torchvision's file for t; returns its size."""
    want = pil_pixels(torchvision_file(t))
    px, info = read_png(data)
    assert info["ctype"] == 2 and info["zlib_header"] == b"\x78\x9c"
    assert np.array_equal(px, want)
    assert np.array_equal(pil_pixels(data), want)
    H, W = want.shape[:2]
    assert info["n_idat"] == len(png.segment_plan(H, W))
    return len(data)


SHAPES = [(3, 1, 1), (3, 1, 37), (3, 23, 1), (3, 5, 3), (3, 17, 33), (3, 64, 257), (1, 29, 101),
          (3, 50, 1000),     # 150050 filtered bytes: segment boundaries inside rows
          (3, 300, 731)]     # 658200 bytes over 11 segments


@pytest.mark.parametrize("shape", SHAPES)
def test_pixels_equal_torchvision(shape):
    g = torch.Generator().manual_seed(sum(shape))
    t = torch.rand(*shape, generator=g)
    t[:, : shape[1] // 2] = (t[:, : shape[1] // 2] * 4).floor() / 4   # flat areas and repeats next to noise
    data, = png.encode_png([t.cuda()])
    check_file(data, t)


def boundary_values():
    k = np.arange(256, dtype=np.float32)
    v = np.concatenate([k / 255, (k + 0.5) / 255, np.float32([-1, -1e-8, -0.0, 0.0, 1.0, 1 + 1e-7, 2, 255, 1e30, -1e30])])
    v = np.concatenate([v, np.nextafter(v, np.float32(np.inf)), np.nextafter(v, np.float32(-np.inf))]).astype(np.float32)
    return torch.from_numpy(v)


@pytest.mark.parametrize("C", [1, 3])
def test_quantisation_boundaries(C):
    v = boundary_values()
    n = v.numel()
    t = torch.cat([v, v.flip(0)])[: (2 * n // C) * C].view(C, 1, -1).expand(C, 3, -1).contiguous()
    data, = png.encode_png([t.cuda()])
    check_file(data, t)


@pytest.mark.parametrize("C", [1, 3])
def test_constant_images_match_across_segments(C):
    for val in (0.0, 0.5, 1.0):
        t = torch.full((C, 400, 1111), val)
        data, = png.encode_png([t.cuda()])
        n = check_file(data, t)
        assert n < png.stream_bytes(400, 1111) / 50   # long matches reaching back over segment boundaries


def test_noise_falls_back_to_stored_blocks():
    t = torch.rand(3, 1024, 1024, generator=torch.Generator().manual_seed(5))
    data, = png.encode_png([t.cuda()])
    n = check_file(data, t)
    raw = 3 * 1024 * 1024
    assert n <= raw * 1.01 + 1024


def test_batched_call_is_byte_equal_to_single_calls():
    g = torch.Generator().manual_seed(11)
    imgs = [torch.rand(3, 1, 1, generator=g), torch.rand(1, 70, 999, generator=g), torch.zeros(3, 200, 300),
            (torch.rand(3, 128, 640, generator=g) * 8).floor() / 8, torch.rand(3, 9, 13, generator=g)]
    dev = [t.cuda() for t in imgs]
    batched = png.encode_png(dev)
    single = [png.encode_png([t])[0] for t in dev]
    assert batched == single
    for d, t in zip(batched, imgs):
        check_file(d, t)
    assert png.encode_png(dev) == batched   # and from run to run


def test_uint8_images_are_taken_as_they_are():
    a = torch.randint(0, 256, (3, 31, 45), dtype=torch.uint8, generator=torch.Generator().manual_seed(2))
    for rule in png.RULES:
        data, = png.encode_png([a.cuda()], rule)
        assert np.array_equal(read_png(data)[0], a.permute(1, 2, 0).numpy())


def test_rejections():
    with pytest.raises(ValueError):
        png.encode_png([torch.zeros(2, 4, 4, device="cuda")])
    with pytest.raises(ValueError):
        png.encode_png([torch.zeros(3, 4, 4, device="cuda", dtype=torch.float64)])
    with pytest.raises(ValueError):
        png.encode_png([torch.zeros(3, 4, 8, device="cuda")[:, :, ::2]])


@pytest.mark.parametrize("kind", ["mnist", "rgb"])
def test_canvas_and_size_against_pil(kind, capsys):
    t = (mnist_canvas if kind == "mnist" else rgb_canvas)(seed=3)
    assert tuple(t.shape) == (3, 3840, 1920)
    data, = png.encode_png([t.cuda()])
    n = check_file(data, t)
    pil = len(torchvision_file(t))
    with capsys.disabled():
        print(f"\n{kind} canvas: GPU {n} bytes, PIL {pil} bytes, ratio {n / pil:.3f}")
    assert n <= 1.5 * pil


def test_save_image_paths(tmp_path):
    t = torch.rand(4, 1, 20, 30, generator=torch.Generator().manual_seed(4))
    png.save_image(t.cuda(), str(tmp_path / "gpu.png"), nrow=2, padding=3)
    vutils.save_image(t, str(tmp_path / "cpu.png"), nrow=2, padding=3)
    a, b = (open(tmp_path / f, "rb").read() for f in ("gpu.png", "cpu.png"))
    assert a != b and np.array_equal(read_png(a)[0], pil_pixels(b))
    buf = io.BytesIO()
    png.save_image(t.cuda(), buf, format="png", nrow=2, padding=3)
    assert buf.getvalue() == a
    nan = t.clone()
    nan[0, 0, 0, 0] = float("nan")
    png.save_image(nan.cuda(), str(tmp_path / "nan.png"))   # torchvision's path: whatever it writes, unchanged
    vutils.save_image(nan, str(tmp_path / "nan_cpu.png"))
    assert open(tmp_path / "nan.png", "rb").read() == open(tmp_path / "nan_cpu.png", "rb").read()


class _Rec:
    def __init__(self):
        self.summaries = []

    def add_summary(self, s, step=None, walltime=None):
        self.summaries.append((s, step))


def _records(writer, *args, **kw):
    rec = _Rec()
    writer._get_file_writer = lambda: rec
    writer.add_image(*args, **kw)
    (s, step), = rec.summaries
    v, = s.value
    return v.tag, step, v.image


@pytest.mark.parametrize("case", ["chw_np", "hwc_cuda", "u8_np", "nan_np", "grey_np"])
def test_tensorboard_image_matches_the_base_writer(tmp_path, monkeypatch, case):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    monkeypatch.syspath_prepend(os.path.join(root, "dropin"))
    monkeypatch.delitem(sys.modules, "tensorboardX", raising=False)
    import tensorboardX
    Base = [c for c in tensorboardX.SummaryWriter.__mro__ if c.__module__.startswith(("torch.", "tensorboardX."))][-1]
    assert "add_image" in vars(tensorboardX.SummaryWriter)
    g = np.random.RandomState(7)
    x = (g.rand(3, 37, 53) * 1.4 - 0.2).astype(np.float32)
    x[:, :5] = boundary_values()[: 5 * 53].view(5, 53).numpy()
    kw = {}
    if case == "hwc_cuda":
        x, kw = torch.from_numpy(x.transpose(1, 2, 0).copy()).cuda(), dict(dataformats="HWC")
    elif case == "u8_np":
        x = (g.rand(3, 37, 53) * 255).astype(np.uint8)
    elif case == "nan_np":
        x[0, 0, 0] = np.nan
    elif case == "grey_np":
        x = x[:1]
    ours = _records(tensorboardX.SummaryWriter(str(tmp_path / "a")), "tag/x", x, 12, **kw)
    base = _records(Base(str(tmp_path / "b")), "tag/x", x.cpu() if torch.is_tensor(x) else x, 12, **kw)
    assert ours[:2] == base[:2]
    for f in ("height", "width", "colorspace"):
        assert getattr(ours[2], f) == getattr(base[2], f)
    a, b = ours[2].encoded_image_string, base[2].encoded_image_string
    assert np.array_equal(np.asarray(Image.open(io.BytesIO(a))), np.asarray(Image.open(io.BytesIO(b))))
    if case in ("chw_np", "hwc_cuda", "u8_np"):
        assert a != b   # encoded on the GPU
        assert np.array_equal(read_png(a)[0], np.asarray(Image.open(io.BytesIO(b))))
    else:
        assert a == b   # the base writer's own record


@pytest.mark.parametrize("case", ["d64_c1_eq", "d64_c3_below"])
def test_vis_seq_png_equals_torchvision(tmp_path, monkeypatch, case):
    """vis_seq with the drop-in's PNG writer writes the same file names as with torchvision's, with equal pixels."""
    from p2pvg_b200 import visualize as V
    from tests.test_generate_engine_gpu import precision
    from tests.test_vis_gpu import FIX, fixture_model, inject_eps
    from tests.vis_ref import Recorder, case_input
    c = next(c for c in torch.load(FIX, weights_only=False)["cases"] if c["case"] == case)
    sp = c["spec"]
    files = {}
    for name, save in (("torchvision", None), ("gpu", png.save_image)):
        r = Recorder()
        monkeypatch.setitem(sys.modules, "imageio", r.imageio)
        d = tmp_path / name
        (d / "gen_vis").mkdir(parents=True)
        with precision("fp32"):
            model = fixture_model(c)
            model.opt.log_dir = str(d)
            inject_eps(monkeypatch, c["eps"])
            np.random.seed(c["np_seed"])
            V.vis_seq(model, case_input(sp).cuda(), 7, sp["L"], model_mode=sp["mode"], recon_mode=sp["recon"],
                      skip_frame=sp["skip"], writer=r, opt=model.opt, save_png=save)
        files[name] = {f: open(d / "gen_vis" / f, "rb").read() for f in os.listdir(d / "gen_vis")}
    assert sorted(files["gpu"]) == sorted(files["torchvision"]) and len(files["gpu"]) == 1
    for f, data in files["gpu"].items():
        assert data != files["torchvision"][f]
        want = pil_pixels(files["torchvision"][f])
        assert np.array_equal(read_png(data)[0], want) and np.array_equal(pil_pixels(data), want)
