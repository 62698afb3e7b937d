"""Moving MNIST host side (no GPU): the MNIST idx reader / resize of load_mnist_digits and the drop-in data package wiring."""
import gzip
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from PIL import Image

from p2pvg_b200.data import load_mnist_digits

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def write_idx(path, imgs, gz=False):
    n, r, c = imgs.shape
    raw = (0x803).to_bytes(4, "big") + b"".join(v.to_bytes(4, "big") for v in (n, r, c)) + imgs.astype(np.uint8).tobytes()
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with (gzip.open if gz else open)(path, "wb") as f:
        f.write(raw)


def synthetic_mnist(n, seed):
    return np.random.RandomState(seed).randint(0, 256, (n, 28, 28)).astype(np.uint8)


@pytest.mark.parametrize("gz", [False, True])
@pytest.mark.parametrize("train", [True, False])
def test_load_mnist_digits_equals_pil_bilinear(tmp_path, gz, train):
    imgs = synthetic_mnist(7, seed=int(gz) + 2 * int(train))
    name = ("train" if train else "t10k") + "-images-idx3-ubyte" + (".gz" if gz else "")
    write_idx(str(tmp_path / "MNIST" / "raw" / name), imgs, gz=gz)
    got = load_mnist_digits(str(tmp_path), train=train)
    assert got.dtype == torch.uint8 and tuple(got.shape) == (7, 32, 32)
    for i, a in enumerate(imgs):
        want = np.asarray(Image.fromarray(a).resize((32, 32), Image.BILINEAR))
        assert np.array_equal(got[i].numpy(), want), i


def test_load_mnist_digits_missing_file_names_the_path(tmp_path):
    with pytest.raises(FileNotFoundError, match=os.path.join("MNIST", "raw", "t10k-images-idx3-ubyte")):
        load_mnist_digits(str(tmp_path), train=False)


def test_load_mnist_digits_rejects_a_truncated_file(tmp_path):
    p = tmp_path / "MNIST" / "raw" / "train-images-idx3-ubyte"
    write_idx(str(p), synthetic_mnist(3, seed=0))
    p.write_bytes(p.read_bytes()[:-5])
    with pytest.raises(ValueError):
        load_mnist_digits(str(tmp_path))


def run_dropin(code, ref):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.join(ROOT, "dropin"), ROOT]), P2PVG_REF=ref)
    return subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, cwd="/")


def test_dropin_data_utils_overrides_only_the_mnist_branches():
    code = ("import data.data_utils as du; assert du.load_dataset.__module__ == 'data.data_utils'\n"
            "try:\n    du.get_generator\nexcept ImportError:\n    print('ok')")
    out = run_dropin(code, ref="")   # no reference checkout: the mnist path still imports, delegation says what is missing
    assert out.returncode == 0 and "ok" in out.stdout, out.stderr


def test_dropin_data_utils_delegates_to_the_reference():
    ref = os.environ.get("P2PVG_REF", "")
    if not ref or not os.path.isfile(os.path.join(ref, "data", "data_utils.py")):
        pytest.skip("P2PVG_REF does not name a reference checkout")
    code = ("import os, data.data_utils as du, data.moving_mnist as mm; "
            "assert os.path.samefile(du.get_generator.__code__.co_filename, os.path.join(os.environ['P2PVG_REF'], 'data', 'data_utils.py')); "
            "assert hasattr(mm, 'DynamicLengthMovingMNIST'); print('ok')")
    out = run_dropin(code, ref=ref)
    assert out.returncode == 0 and "ok" in out.stdout, out.stderr
