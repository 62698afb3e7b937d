"""Float64 statements the launch tests of every backbone check kernels against (tests/test_*launches_gpu.py): GEMM references
on strided operands, exact sums of 0 / 1 products, element-wise bounds, BatchNorm statistics and the BatchNorm backward of
one group.

The checkers work in chunks of CHUNK elements so that float64 references of benchmark-sized tensors (up to 10^9 elements)
stay a few GiB.
"""
import torch

from p2pvg_b200.engine import ACT_LRELU

CHUNK = 1 << 25     # elements of one float64 chunk (256 MB)
A_STAT = 2.0 ** -18   # a statistics row: a fixed-order fp32 tree over 128 stored values (see test_tc_schedule_gpu.py)
EPS = 1e-5


# ------------------------------------------------------------------ exact reductions

def binary01(shape, p=0.25):
    """bf16 0 / 1 operand, 1 with probability p.  Products are 0 / 1 and a K-long sum of them is an integer <= K: below 2^24 every
    fp32 partial sum is exact in any order, so a kernel's result must equal the float64 reference bit for bit."""
    return (torch.rand(*shape, device="cuda") < p).to(torch.bfloat16)


def assert_exact(got, ref, K, name):
    """The fp32 result of a reduction of 0 / 1 products over K < 2^24 terms equals float64 exactly."""
    assert K < 1 << 24, f"{name}: K = {K} is too long for exact fp32 integer sums"
    bad = got.double() != ref
    if bad.any():
        i = tuple(int(v) for v in torch.unravel_index(torch.nonzero(bad.flatten())[0, 0], got.shape))
        raise AssertionError(f"{name}: {int(bad.sum())}/{bad.numel()} elements differ from the exact integer sum, first at {i}: "
                             f"got {got[i].item():.9g}, exact {ref[i].item():.9g}")
    print(f"[exact] {name}: K={K}, largest sum {ref.max().item():.0f}, exact")


def bound_check(got, ref, bound, name):
    """|got - ref| <= bound element-wise (float64 ref and bound); returns the worst ratio."""
    diff = (got.double() - ref).abs()
    ratio = torch.where(bound > 0, diff / bound.clamp_min(1e-300), torch.where(diff > 0, torch.inf, 0.0))
    ratio = torch.nan_to_num(ratio, nan=torch.inf)
    worst = ratio.max().item()
    if worst > 1.0:
        i = int(ratio.argmax())
        raise AssertionError(f"{name}: worst ratio {worst:.3g} at {i}: got {got.flatten()[i].item():.8g}, "
                             f"ref {ref.flatten()[i].item():.8g}, bound {bound.flatten()[i].item():.3g}")
    return worst


# ------------------------------------------------------------------ GEMM (p2pvg_gemm)

def gemm_ref64(A, B, M, N, Kd, a_mn, b_mn, lda, ldb, bias=None, addend=None, ldd=None, c0=None, rows=None):
    """C = opA(A) opB(B) + bias + addend + c0 in float64 (and over |.|) on strided views of the operands, chunked over M and K.
    rows = (m0, m1): only those rows of C (addend and c0 are then those rows too)."""
    Av = A.as_strided((Kd, M), (lda, 1)) if a_mn else A.as_strided((M, Kd), (lda, 1))
    if rows is not None:
        Av = Av[:, rows[0]:rows[1]] if a_mn else Av[rows[0]:rows[1]]
        M = rows[1] - rows[0]
    Bv = B.as_strided((Kd, N), (ldb, 1)) if b_mn else B.as_strided((N, Kd), (ldb, 1))
    ref = torch.zeros(M, N, dtype=torch.float64, device=A.device)
    absref = torch.zeros_like(ref)
    mc = max(1, min(M, CHUNK // max(1, min(Kd, 4096))))
    kc = max(1, min(Kd, CHUNK // max(mc, N)))
    for m0 in range(0, M, mc):
        for k0 in range(0, Kd, kc):
            a = (Av[k0:k0 + kc, m0:m0 + mc].t() if a_mn else Av[m0:m0 + mc, k0:k0 + kc]).double()
            b = (Bv[k0:k0 + kc] if b_mn else Bv[:, k0:k0 + kc].t()).double()
            ref[m0:m0 + mc] += a @ b
            absref[m0:m0 + mc] += a.abs() @ b.abs()
    for extra in (bias, addend, c0):
        if extra is not None:
            e = extra.double()
            ref += e
            absref += e.abs()
    return ref, absref


# ------------------------------------------------------------------ BatchNorm

def finalize_ref(s1, s2, m1, R, gamma, beta, eps, a_rel):
    """Float64 mean / invstd / var_unbiased / scale / shift of groups whose sums are (s1, s2) with magnitudes (m1 = sum|x|,
    s2 = sum x^2), each sum known within a_rel of its magnitude; returns [(ref, bound)] in the kernel's output order."""
    E1, E2 = m1 / R, s2 / R
    m = s1 / R
    var = (s2 / R - m * m).clamp_min(0.0)
    g, bt = gamma.double(), beta.double()
    invstd = 1.0 / torch.sqrt(var + eps)
    u = 2.0 ** -23
    d_m = a_rel * E1 + u * m.abs()
    d_var = 3.0 * a_rel * E2 + u * var
    d_is = invstd * (0.5 * d_var / (var + eps) * 1.01 + u)
    sc = g * invstd
    d_sc = g.abs() * d_is + u * sc.abs()
    sh = bt - m * sc
    d_sh = m.abs() * d_sc + sc.abs() * d_m + u * (bt.abs() + (m * sc).abs()) * 2
    varu = var * R / (R - 1)
    return [(m, d_m), (invstd, d_is), (varu, d_var * R / (R - 1) + u * varu), (sc, d_sc), (sh, d_sh)]


def check_finalize_vs_output(K, part, parts_per_group, out, G, rows_per_group, Cn, name=""):
    """bn_fwd_finalize_tiles with the engine's parts_per_group against float64 statistics of the stored output."""
    gamma = torch.rand(Cn, device=out.device) + 0.5
    beta = torch.randn(Cn, device=out.device)
    outs = [torch.empty(G * Cn, device=out.device) for _ in range(5)]
    K.bn_fwd_finalize_tiles(part, parts_per_group, Cn, 1, G, rows_per_group, Cn, gamma, beta, *outs)
    flat = out.reshape(G, rows_per_group, Cn)
    s1 = torch.empty(G, Cn, dtype=torch.float64, device=out.device)
    s2, m1 = torch.empty_like(s1), torch.empty_like(s1)
    per = max(1, CHUNK // Cn)
    for g in range(G):
        a = b = c = 0.0
        for r0 in range(0, rows_per_group, per):
            x = flat[g, r0:r0 + per].double()
            a, b, c = a + x.sum(0), b + (x * x).sum(0), c + x.abs().sum(0)
        s1[g], s2[g], m1[g] = a, b, c
    worst = 0.0
    for got, (ref, bound), nm in zip(outs, finalize_ref(s1, s2, m1, rows_per_group, gamma, beta, 1e-5, A_STAT),
                                     ("mean", "invstd", "var_unbiased", "scale", "shift")):
        worst = max(worst, bound_check(got.view(G, Cn), ref, bound, f"{name} finalize {nm}"))
    print(f"[bound] {name} finalize ({G} groups x {parts_per_group} parts): worst error/bound {worst:.3g}")
    return worst


def bn_group_ref64(x, dy, gamma, beta, act, side=None, y=None):
    """Float64 training-mode BatchNorm of one group x [R, C] followed by `act`: statistics, dz = dy * act'(pre), and
    dx = gamma invstd (dz - mean dz - xhat mean(dz xhat)) with its magnitude.  LeakyReLU: `side` is the slope side the kernel
    uses (sign of its fp32 fmaf); tanh: 1 - y^2 of the stored y."""
    x = x.double()
    R = x.shape[0]
    m = x.mean(0)
    v = ((x - m) ** 2).mean(0)
    inv = 1.0 / torch.sqrt(v + EPS)
    xh = (x - m) * inv
    if dy is None:
        return dict(mean=m, var=v, invstd=inv, xhat=xh)
    if act == ACT_LRELU:
        dz = dy.double() * torch.where(side, 1.0, 0.2)
    else:
        dz = dy.double() * (1 - y.double() ** 2)
    sdz, sdzx = dz.sum(0), (dz * xh).sum(0)
    k0 = gamma.double() * inv
    dx = k0 * (dz - sdz / R - xh * sdzx / R)
    mag = k0.abs() * (dz.abs() + (dz.abs().sum(0) + xh.abs() * (dz * xh).abs().sum(0)) / R)
    return dict(mean=m, var=v, invstd=inv, dz=dz, sdz=sdz, sdzx=sdzx, dx=dx, dx_mag=mag, sdz_mag=dz.abs().sum(0),
                sdzx_mag=(dz * xh).abs().sum(0))
