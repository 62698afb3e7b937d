"""The float64 statements of tests/gen_audit.py reject what they must: fp32 emulations of p2pvg_lstm_step, p2pvg_pose_mlp and
bn_eval_coeffs + the folded eval epilogue pass them, and the same emulations with one deliberate corruption each (the gate
order, the counter_rows group, the decoder's skip row, the shift without mean * scale, LayerNorm with the unbiased variance)
are rejected."""
import pytest
import torch

from p2pvg_b200.models.h36m_mlp import decoder, encoder
from tests.gen_audit import (bn_coeffs64, bn_module64, embed64, fold_bound, head_gauss64, head_tanh64, lstm_cell64, lstm_input64,
                             pose_decoder64, residual64, residual_params)
from tests.ref64 import bound_check


def _rejects(fn):
    with pytest.raises(AssertionError):
        fn()


# ------------------------------------------------------------------ p2pvg_lstm_step

def _lstm_case(seed=0, rows=21, R=64, ga=24, gb=8, G=3):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, sc=1.0: sc * torch.randn(*s, generator=g)
    in_dim = ga + gb + 2
    return dict(rows=rows, R=R, ga=ga, gb=gb, G=G, seg_a=r(3 * rows * ga), seg_b=r(2 * rows * gb), ia=2, ib=1,
                tuc=torch.rand(G, generator=g), dt=torch.rand(G, generator=g) + 1, counter_rows=rows // G,
                w_e=r(R, in_dim, sc=0.2), b_e=r(R, sc=0.1), w_ih=r(4 * R, R, sc=0.15), b_ih=r(4 * R, sc=0.1),
                w_hh=r(4 * R, R, sc=0.15), b_hh=r(4 * R, sc=0.1), h0=r(rows, R, sc=0.5), c0=r(rows, R), w_o=r(10, R, sc=0.2),
                b_o=r(10, sc=0.1), w_o2=r(10, R, sc=0.2), b_o2=r(10, sc=0.1), eps=r(rows, 10))


def _lstm_emulate(c, gate_order=(0, 1, 2, 3), group=None):
    """lstm_step.cu in fp32 (one module, one layer, gaussian head).  gate_order: the chunks read as (i, f, g, o); group(b):
    the counter group of row b (default b // counter_rows)."""
    rows, ga, gb, R = c["rows"], c["ga"], c["gb"], c["R"]
    a = c["seg_a"][c["ia"] * rows * ga:(c["ia"] + 1) * rows * ga].view(rows, ga)
    b = c["seg_b"][c["ib"] * rows * gb:(c["ib"] + 1) * rows * gb].view(rows, gb)
    grp = torch.tensor([group(i) if group else i // c["counter_rows"] for i in range(rows)])
    X = torch.cat([a, b, c["tuc"][grp][:, None], c["dt"][grp][:, None]], 1)
    e = X @ c["w_e"].t() + c["b_e"]
    pre = (e @ c["w_ih"].t() + c["b_ih"]) + (c["h0"] @ c["w_hh"].t() + c["b_hh"])
    ch = [pre[:, k * R:(k + 1) * R] for k in gate_order]
    i, f, gg, o = torch.sigmoid(ch[0]), torch.sigmoid(ch[1]), torch.tanh(ch[2]), torch.sigmoid(ch[3])
    cc = f * c["c0"] + i * gg
    h = o * torch.tanh(cc)
    mu, lv = h @ c["w_o"].t() + c["b_o"], h @ c["w_o2"].t() + c["b_o2"]
    return h, cc, c["eps"] * torch.exp(0.5 * lv) + mu


def _lstm_check(c, h, cc, out):
    X = lstm_input64(c["seg_a"], c["ia"], c["ga"], c["seg_b"], c["ib"], c["gb"], c["tuc"], c["dt"], c["counter_rows"], c["rows"])
    x, xe = embed64(X, c["w_e"], c["b_e"])
    hr, cr, eh, ec = lstm_cell64(x, xe, c["h0"], c["c0"], c["w_ih"], c["b_ih"], c["w_hh"], c["b_hh"])
    bound_check(cc, cr, ec, "c")
    bound_check(h, hr, eh, "h")
    ref, e = head_gauss64(h.double(), c["w_o"], c["b_o"], c["w_o2"], c["b_o2"], c["eps"])
    bound_check(out, ref, e, "head")


def test_lstm_step_emulation_passes():
    c = _lstm_case()
    _lstm_check(c, *_lstm_emulate(c))


def test_lstm_step_wrong_gate_order_rejected():
    c = _lstm_case(1)
    _rejects(lambda: _lstm_check(c, *_lstm_emulate(c, gate_order=(0, 1, 3, 2))))   # (i, f, o, g): PyTorch's order is (i, f, g, o)
    _rejects(lambda: _lstm_check(c, *_lstm_emulate(c, gate_order=(1, 0, 2, 3))))


def test_lstm_step_wrong_counter_group_rejected():
    c = _lstm_case(2)
    _rejects(lambda: _lstm_check(c, *_lstm_emulate(c, group=lambda b: b % c["G"])))
    _rejects(lambda: _lstm_check(c, *_lstm_emulate(c, group=lambda b: 0)))


def test_lstm_head_tanh():
    c = _lstm_case(3)
    h = torch.tanh(c["h0"])
    y = torch.tanh(h @ c["w_o"].t() + c["b_o"])
    ref, e = head_tanh64(h.double(), c["w_o"], c["b_o"])
    bound_check(y, ref, e, "tanh head")
    _rejects(lambda: bound_check(torch.tanh(h @ c["w_o"].t()), ref, e, "tanh head without bias"))


# ------------------------------------------------------------------ p2pvg_pose_mlp

def _perturbed(mod, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for p in mod.parameters():
            p.add_(0.1 * torch.randn(p.shape, generator=g))
    return mod


def _residual_emulate(rl, x, unbiased=False):
    sc = torch.relu(x @ rl.shortcut[0].weight.t() + rl.shortcut[0].bias)
    a = x
    for k in (0, 2, 4):
        a = torch.relu(a @ rl.long_path[k].weight.t() + rl.long_path[k].bias)
    y = sc + a
    m = y.mean(1, keepdim=True)
    v = y.var(1, unbiased=unbiased, keepdim=True)
    return (y - m) / torch.sqrt(v + 1e-5) * rl.norm.weight + rl.norm.bias


@pytest.mark.parametrize("g", [32, 128])
def test_pose_residual_emulation_passes_unbiased_variance_rejected(g):
    """fc1 of the encoder (51 -> g, a 25-unit long path) and fc2 (g -> g)."""
    enc = _perturbed(encoder(51, g, g), g)
    x = 3 * torch.randn(21, 51, generator=torch.Generator().manual_seed(g))
    with torch.no_grad():
        for rl, xin in ((enc.fc1, x), (enc.fc2, torch.randn(21, g))):
            ref, e = residual64(residual_params(rl), xin.double(), None)
            bound_check(_residual_emulate(rl, xin), ref, e, "residual")
            _rejects(lambda: bound_check(_residual_emulate(rl, xin, unbiased=True), ref, e, "residual, unbiased variance"))


def test_pose_decoder_skip_row_modulo():
    """Output row r reads skip row r % nsrc: the emulation that reads row r is rejected (the skip buffers hold more rows
    than nsrc, as an encode of the whole clip does)."""
    g, rows, nsrc = 32, 21, 7
    dec = _perturbed(decoder(g, 51, g), 7)
    gen = torch.Generator().manual_seed(8)
    vec, s1, s2 = torch.randn(rows, g, generator=gen), torch.randn(rows, g, generator=gen), torch.randn(rows, g, generator=gen)

    def emulate(row):
        r = torch.tensor([row(i) for i in range(rows)])
        d1 = _residual_emulate(dec.fc1, vec)
        d2 = _residual_emulate(dec.fc2, torch.cat([d1, s2[r]], 1))
        return torch.cat([d2, s1[r]], 1) @ dec.fc3.weight.t() + dec.fc3.bias

    with torch.no_grad():
        ref, e = pose_decoder64(dec, vec, s1[:nsrc], s2[:nsrc], nsrc)
        bound_check(emulate(lambda r: r % nsrc), ref, e, "decoder")
        _rejects(lambda: bound_check(emulate(lambda r: r), ref, e, "decoder reading skip row r"))
        # and the reference itself, told to read row r, disagrees with the kernel's r % nsrc
        ref_r, e_r = pose_decoder64(dec, vec, s1, s2, nsrc, skip_row=lambda r, n: r)
        _rejects(lambda: bound_check(emulate(lambda r: r % nsrc), ref_r, e_r, "reference reading skip row r"))


# ------------------------------------------------------------------ bn_eval_coeffs and the folded epilogue

def _bn_case(C=64, seed=0):
    g = torch.Generator().manual_seed(seed)
    gamma_, beta = 1 + 0.2 * torch.randn(C, generator=g), 0.1 * torch.randn(C, generator=g)
    mean, var = 0.1 * torch.randn(C, generator=g), 0.5 + torch.rand(C, generator=g)
    var[:4] = 1e-3
    mean[:4] = torch.tensor([4.0, -4.0, 8.0, -8.0])   # |mean| >= 100 sqrt(var)
    return gamma_, beta, mean, var


def test_bn_eval_coeffs_emulation_passes_missing_mean_term_rejected():
    gamma_, beta, mean, var = _bn_case()
    sc = gamma_ / torch.sqrt(var + 1e-5)
    ref_sc, ref_sh, e_sc, e_sh = bn_coeffs64(gamma_, beta, mean, var, 1e-5)
    bound_check(sc, ref_sc, e_sc, "scale")
    bound_check(beta - mean * sc, ref_sh, e_sh, "shift")
    _rejects(lambda: bound_check(beta, ref_sh, e_sh, "shift without mean * scale"))
    # the corrupted statement (shift without mean * scale) rejects the correct kernel
    _, bad_sh, _, bad_e = bn_coeffs64(gamma_, beta, mean, var, 1e-5, with_shift_term=False)
    _rejects(lambda: bound_check(beta - mean * sc, bad_sh, bad_e, "correct shift against the corrupted statement"))


def test_folded_epilogue_against_module_formula():
    """fmaf(x, scale, shift) in fp32 against (x - mean) / sqrt(var + eps) gamma + beta within fold_bound, x spread around each
    channel's mean (where the fold cancels); the fold of a shift without mean * scale is rejected."""
    gamma_, beta, mean, var = _bn_case(seed=1)
    x = (mean + torch.sqrt(var) * torch.randn(4096, 64, generator=torch.Generator().manual_seed(2))).float()
    sc = gamma_ / torch.sqrt(var + 1e-5)
    sh = beta - mean * sc
    got = torch.addcmul(sh, x, sc)
    ref = bn_module64(x, gamma_, beta, mean, var, 1e-5)
    b = fold_bound(x, gamma_, beta, mean, var, 1e-5)
    w = bound_check(got, ref, b, "folded eval BatchNorm")
    assert w > 1e-3, "the bound is so loose that the emulation's error does not show against it"
    _rejects(lambda: bound_check(torch.addcmul(beta, x, sc), ref, b, "fold without mean * scale"))
