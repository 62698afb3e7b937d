"""p2pvg_gif_encode on the GPU: every file decodes with PIL and with tests/gif_ref.py to the same frames, delays and loop;
frames of at most 256 colours exactly, others within Pillow's adaptive-palette error; every frame's LZW data equals the
host restatement's coding of its index map."""
import io
import os
import struct
import sys

import numpy as np
import pytest
import torch
from PIL import Image

from p2pvg_b200 import gif
from tests.gif_ref import encode_frame_data, frame_stream_bytes, read_gif
from tests.test_gif_cpu import dropin  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu


def pil_decode(data):
    im = Image.open(io.BytesIO(data))
    out, durations = [], []
    for k in range(im.n_frames):
        im.seek(k)
        out.append(np.asarray(im.convert("RGB")))
        durations.append(im.info.get("duration"))
    return np.stack(out), durations, im.info.get("loop")


def mse(a, b):
    return float(((a.astype(np.float64) - b.astype(np.float64)) ** 2).mean())


def pillow_mse(frame):
    q = Image.fromarray(frame).convert("P", palette=Image.ADAPTIVE, colors=256)
    return mse(np.asarray(q.convert("RGB")), frame)


def check_file(data, frames, delay_cs=10):
    """data decodes with both readers to the same frames, delay and loop 0; frames [T, H, W, 3] uint8 of at most 256
    colours decode exactly, others within Pillow's adaptive-palette MSE + 0.01; each frame's LZW data is the host
    restatement's coding of its index map.  Returns the decoded frames."""
    got, info = read_gif(data)
    pil, durations, loop = pil_decode(data)
    assert np.array_equal(got, pil)
    assert got.shape == frames.shape
    assert info["loop"] == loop == 0
    assert info["delays"] == [delay_cs] * len(frames) and durations == [10 * delay_cs] * len(frames)
    assert info["min_sizes"] == [8] * len(frames)
    for t, f in enumerate(frames):
        n_col = len(np.unique(f.reshape(-1, 3), axis=0))
        if n_col <= 256:
            assert np.array_equal(got[t], f), f"frame {t} of {n_col} colours is not lossless"
        else:
            assert mse(got[t], f) <= pillow_mse(f) + 0.01
    for idx, body, sizes in zip(info["indices"], frame_stream_bytes(data), info["block_sizes"]):
        assert body == encode_frame_data(idx)
        assert all(s == 255 for s in sizes[:-1])
    return got


def encode1(frames, **kw):
    data, = gif.encode_gif([torch.from_numpy(np.ascontiguousarray(frames)).cuda()], **kw)
    return data


def grey_digits(T, H, W, seed):
    g = np.random.RandomState(seed)
    f = np.zeros((T, H, W), np.uint8)
    for t in range(T):
        for _ in range(3):
            y, x = g.randint(0, max(1, H - 12)), g.randint(0, max(1, W - 12))
            f[t, y:y + 12, x:x + 12] = g.randint(0, 256, (min(12, H - y), min(12, W - x)))
    return np.repeat(f[..., None], 3, 3)


def smooth_colour(T, H, W, seed):
    g = np.random.RandomState(seed)
    y, x = np.mgrid[:H, :W].astype(np.float64)
    out = []
    for t in range(T):
        r = 128 + 100 * np.sin(x / 37 + t) * np.cos(y / 23)
        gg = 128 + 100 * np.sin((x + y) / 51 - t)
        b = 128 + 100 * np.cos(x / 19 - y / 31 + t)
        out.append(np.stack([r, gg, b], -1) + g.randint(-6, 7, (H, W, 3)))
    return np.clip(np.stack(out), 0, 255).astype(np.uint8)


def with_borders(frames):
    f = frames.copy()
    f[:, :2] = (255, 165, 0)   # orange
    f[:, -2:] = (255, 0, 0)    # red
    return f


LOSSLESS = {
    "one_colour": lambda: np.full((3, 20, 30, 3), (12, 200, 99), np.uint8),
    "exactly_256": lambda: np.random.RandomState(1).permutation(
        np.stack([np.arange(256), (np.arange(256) * 7) % 256, 255 - np.arange(256)], 1))[
        np.random.RandomState(2).randint(0, 256, 2 * 64 * 48)].reshape(2, 64, 48, 3).astype(np.uint8),
    "grey_mnist": lambda: grey_digits(4, 64, 384, 5),
    "pixel": lambda: np.full((2, 1, 1, 3), 77, np.uint8),
    "row": lambda: grey_digits(2, 12, 65535, 6)[:, :1],
    "column": lambda: grey_digits(2, 65535, 12, 7)[:, :, :1],
    "many_segments_full_table": lambda: np.random.RandomState(3).randint(0, 256, (2, 400, 420, 1)).repeat(3, 3).astype(
        np.uint8),
}


@pytest.mark.parametrize("case", sorted(LOSSLESS))
def test_lossless_frames(case):
    frames = LOSSLESS[case]()
    check_file(encode1(frames), frames)


LOSSY = {
    "colours_257": lambda: np.concatenate([LOSSLESS["exactly_256"]()[:1], np.full((1, 64, 48, 3), 3, np.uint8)], 0)[
        :1].copy(),
    "grey_with_borders_258": lambda: with_borders(np.repeat(np.arange(256, dtype=np.uint8)[None, None, :, None].repeat(
        40, 1), 3, 3)),
    "smooth_colour": lambda: smooth_colour(2, 96, 160, 8),
    "noise": lambda: np.random.RandomState(9).randint(0, 256, (1, 80, 120, 3)).astype(np.uint8),
    "colour_640x384": lambda: smooth_colour(2, 384, 640, 10),
    "colour_1280x768": lambda: smooth_colour(1, 768, 1280, 11),
}


@pytest.mark.parametrize("case", sorted(LOSSY))
def test_lossy_frames_within_pillow(case):
    frames = LOSSY[case]()
    if case == "colours_257":
        frames[0, 0, 0] = (1, 2, 3)   # one colour more than the 256 of the table
    n = [len(np.unique(f.reshape(-1, 3), axis=0)) for f in frames]
    assert min(n) > 256 and (case != "colours_257" or n == [257]) and (case != "grey_with_borders_258" or n == [258])
    check_file(encode1(frames), frames)


def test_compose_frames_are_lossless():
    from p2pvg_b200 import visualize as V
    g = torch.Generator().manual_seed(4)
    store0 = torch.rand(8, 1, 16, 16, generator=g).mul(4).floor().div(4).cuda()
    store1 = torch.rand(20, 1, 16, 16, generator=g).cuda()
    np.random.seed(0)
    tiles = V.plan_tiles(4, 5, 2, 2, lambda t: (0, t * 2), lambda s, t: (1, (s * 5 + t) * 2))
    _, _, frames = V.compose(store0, store1, tiles, 1, 16)
    data, = gif.encode_gif([frames])
    f = frames.cpu().numpy()
    got = check_file(data, f)
    if max(len(np.unique(x.reshape(-1, 3), axis=0)) for x in f) <= 256:
        assert np.array_equal(got, f)


def test_batched_call_equals_single_calls_and_repeats():
    anims = [LOSSLESS["grey_mnist"](), LOSSY["smooth_colour"](), LOSSLESS["pixel"](), LOSSY["noise"]()]
    cuda = [torch.from_numpy(a).cuda() for a in anims]
    f32 = torch.rand(3, 3, 17, 23, generator=torch.Generator().manual_seed(1)).cuda()
    batch = gif.encode_gif(cuda + [f32], delay_cs=7, loop=0)
    assert gif.encode_gif(cuda + [f32], delay_cs=7, loop=0) == batch
    singles = [gif.encode_gif([t], delay_cs=7)[0] for t in cuda + [f32]]
    assert batch == singles
    for a, data in zip(anims, batch):
        check_file(data, a, delay_cs=7)


def test_fp32_tensorboard_rule_equals_host_quantised_uint8():
    g = torch.Generator().manual_seed(2)
    x = (torch.rand(3, 3, 45, 67, generator=g) * 1.4 - 0.2)
    x[:, :, :3] = torch.floor(x[:, :, :3] * 8) / 8
    u8 = (x.numpy() * np.float32(255)).clip(0, 255).astype(np.uint8).transpose(0, 2, 3, 1).copy()
    a, = gif.encode_gif([x.cuda()], "tensorboard")
    b = encode1(u8)
    assert a == b
    check_file(a, u8)


def test_save_gif_writes_the_file(tmp_path):
    frames = LOSSLESS["grey_mnist"]()
    gif.save_gif(str(tmp_path / "a.gif"), torch.from_numpy(frames).cuda())
    gif.save_gif(str(tmp_path / "b.gif"), list(frames))
    a, b = (open(tmp_path / n, "rb").read() for n in ("a.gif", "b.gif"))
    assert a == b
    check_file(a, frames)


def test_save_gif_matches_imageio_timing(tmp_path):
    imageio = pytest.importorskip("imageio")
    frames = LOSSLESS["grey_mnist"]()
    gif.save_gif(str(tmp_path / "ours.gif"), list(frames))
    imageio.mimsave(str(tmp_path / "theirs.gif"), list(frames))
    ours = pil_decode(open(tmp_path / "ours.gif", "rb").read())
    theirs = pil_decode(open(tmp_path / "theirs.gif", "rb").read())
    assert len(ours[0]) == len(theirs[0]) and ours[1] == theirs[1] and ours[2] == theirs[2]


# ---- TensorBoard: the video summary and the native record checksum ----------------------------------------------------
def _writers():
    """(the drop-in SummaryWriter, its base class); the test takes the ``dropin`` fixture."""
    import tensorboardX
    Base = [c for c in tensorboardX.SummaryWriter.__mro__ if c.__module__.startswith(("torch.", "tensorboardX."))][-1]
    return tensorboardX.SummaryWriter, Base


class _Rec:
    def __init__(self):
        self.summaries = []

    def add_summary(self, s, step=None, walltime=None):
        self.summaries.append((s, step))


@pytest.mark.parametrize("case", ["f32_np", "u8_cuda", "f32_colour"])
def test_video_summary(tmp_path, monkeypatch, case, dropin):
    Writer, Base = _writers()
    g = np.random.RandomState(5)
    if case == "f32_np":
        vid = (np.floor(g.rand(1, 4, 3, 24, 40) * 8) / 8 * 1.2 - 0.1).astype(np.float32)
    elif case == "u8_cuda":
        vid = torch.from_numpy(g.randint(0, 256, (1, 3, 3, 16, 16)).astype(np.uint8) // 64 * 64).cuda()
    else:
        vid = np.transpose(smooth_colour(3, 32, 48, 1), (0, 3, 1, 2))[None].astype(np.float32) / 255
    w = Writer(str(tmp_path / "a"))
    rec = _Rec()
    w._get_file_writer = lambda: rec
    w.add_video("model/GenVideo10", vid, 7, fps=2)
    (s, step), = rec.summaries
    v, = s.value
    base_rec = _Rec()
    b = Base(str(tmp_path / "b"))
    b._get_file_writer = lambda: base_rec
    b.add_video("model/GenVideo10", vid.cpu().numpy() if torch.is_tensor(vid) else vid, 7, fps=2)
    (bs, bstep), = base_rec.summaries
    assert (v.tag, step) == (bs.value[0].tag, bstep)
    v_np = vid.cpu().numpy() if torch.is_tensor(vid) else vid
    want = v_np[0].transpose(0, 2, 3, 1)
    want = want if want.dtype == np.uint8 else (want.astype(np.float32) * np.float32(255)).clip(0, 255).astype(np.uint8)
    assert (v.image.height, v.image.width, v.image.colorspace) == (want.shape[1], want.shape[2], 3)
    check_file(v.image.encoded_image_string, want, delay_cs=50)


def test_video_summary_defers_other_input(tmp_path, monkeypatch, dropin):
    Writer, Base = _writers()
    seen = []
    monkeypatch.setattr(Base, "add_video", lambda self, *a, **k: seen.append((a, k)))
    w = Writer(str(tmp_path))
    grey = np.zeros((1, 2, 1, 4, 4), np.float32)
    two = np.zeros((2, 2, 3, 4, 4), np.float32)
    f64 = np.zeros((1, 2, 3, 4, 4), np.float64)
    for v in (grey, two, f64):
        w.add_video("v", v, 1, fps=4)
    w.close()
    assert len(seen) == 3 and all(a[1] is v for (a, _), v in zip(seen, (grey, two, f64)))


def _records(path):
    from tensorboard.compat.tensorflow_stub.pywrap_tensorflow import masked_crc32c
    data, out, p = open(path, "rb").read(), [], 0
    while p < len(data):
        n, = struct.unpack("<Q", data[p:p + 8])
        assert struct.unpack("<I", data[p + 8:p + 12])[0] == masked_crc32c(data[p:p + 8])
        body = data[p + 12:p + 12 + n]
        assert struct.unpack("<I", data[p + 12 + n:p + 16 + n])[0] == masked_crc32c(body)
        out.append(data[p:p + 16 + n])
        p += 16 + n
    return out


def test_event_files_are_byte_identical(tmp_path, monkeypatch, dropin):
    Writer, Base = _writers()
    files = {}
    for name, cls in (("dropin", Writer), ("stock", Base)):
        w = cls(str(tmp_path / name))
        for k in range(3):
            w.add_scalar("loss/kl", 0.25 * k, k, walltime=1000.0 + k)
        w.add_histogram("w", np.arange(-50, 50, dtype=np.float64), 5, walltime=1010.0)
        w.add_image("grey", np.linspace(0, 1, 2 * 9 * 11, dtype=np.float32).reshape(2, 9, 11)[:1], 6, walltime=1011.0)
        w.add_scalar("big", 1.0, 7, walltime=1012.0)
        if name == "dropin":
            rw = w._get_file_writer().event_writer._async_writer._writer
            assert "write" in vars(rw)   # the native checksum is in place
        w.close()
        f, = os.listdir(tmp_path / name)
        files[name] = _records(tmp_path / name / f)
    # the first record (file_version) carries the writer's creation time
    assert len(files["dropin"]) == len(files["stock"]) == 7
    assert files["dropin"][1:] == files["stock"][1:]


@pytest.mark.parametrize("case", ["d64_c1_eq", "d64_c3_below"])
def test_vis_seq_gif(tmp_path, monkeypatch, case):
    """vis_seq with save_gif=gif.save_gif writes a GIF that decodes to the gif tensor it returns; without it imageio's
    mimsave is called with the same frames."""
    from p2pvg_b200 import visualize as V
    from tests.test_generate_engine_gpu import precision
    from tests.test_vis_gpu import FIX, fixture_model, inject_eps
    from tests.vis_ref import Recorder, case_input
    c = next(c for c in torch.load(FIX, weights_only=False)["cases"] if c["case"] == case)
    sp = c["spec"]
    out = {}
    for name, save in (("imageio", None), ("gpu", gif.save_gif)):
        r = Recorder()
        monkeypatch.setitem(sys.modules, "imageio", r.imageio)
        d = tmp_path / name
        (d / "gen_vis").mkdir(parents=True)
        with precision("fp32"):
            model = fixture_model(c)
            model.opt.log_dir = str(d)
            inject_eps(monkeypatch, c["eps"])
            np.random.seed(c["np_seed"])
            _, _, g = V.vis_seq(model, case_input(sp).cuda(), 7, sp["L"], model_mode=sp["mode"], recon_mode=sp["recon"],
                                skip_frame=sp["skip"], writer=r, opt=model.opt, save_gif=save)
        out[name] = (r.gifs, g.cpu().numpy(), d)
    gifs, g_ref, _ = out["imageio"]
    (name, frames), = gifs
    assert np.array_equal(np.stack(frames), g_ref)
    no_gifs, g, d = out["gpu"]
    assert no_gifs == [] and np.array_equal(g, g_ref)
    data = open(os.path.join(d, "gen_vis", os.path.basename(name)), "rb").read()
    check_file(data, g)
