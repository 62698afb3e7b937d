"""Host-side launch decisions of the LSTM scan kernels (p2pvg_lstm_scan_fwd / _bwd), mirrored in Python, plus the
teacher-forced float64 references and the error bounds the scan tests share (tests/test_lstm_scan_gpu.py,
tests/test_lstm_ref_cpu.py).

Four kernel families sit behind the two entry points (lstm_scan.cu:329-343):
  cluster8    lstm_cluster.cu     tf32, R in {64, 128, 256}: slabs of 16*MT rows, one cluster of 8 CTAs per slab, R/8 units per CTA
  cluster16   lstm_cluster512.cu  tf32, R = 512: clusters of 16 CTAs, 32 units per CTA; forward MT from a cost model, backward MT = 1
  coop-tf32   lstm_scan.cu <true>   tf32, any other R (R = 192 in the bf16 engine): cooperative grid of (R/8) x ceil(B/64) CTAs
  coop-exact  lstm_scan.cu <false>  exact fp32 (FFMA chains, libm activations): every R in fp32 mode
A slab (or, cooperatively, a 64-row block) is what one cluster (row of CTAs) owns; `scan_schedule` says which one a batch row
lands in, how full the last one is, and how many waves of resident clusters the launch takes.

The references are teacher-forced: every step is recomputed in float64 from the state the kernel itself stored (hs[s], cs[s],
gates[s], dG[s+1]), so errors do not compound across steps and the bounds stay per-step tight.  The TF32 families round both
operands of the recurrent product with cvt.rna.tf32.f32; `tf32_rna` does the same on the bit pattern, so the reference multiplies
the very operands the tensor cores see and the bound has no operand-conversion term.
"""
import math
from dataclasses import dataclass

import numpy as np
import torch

MT2_ABOVE = 128          # lstm_cluster.cu:397-398 kMt2Above: 32-row slabs above this batch size
COOP_ROWS = 64           # lstm_scan.cu:16 RB
COOP_UNITS = 8           # lstm_scan.cu:15 UB


def cdiv(a, b):
    return (a + b - 1) // b


def max_clusters(lib, R):
    """cudaOccupancyMaxActiveClusters of every instance, by the diagnostics' `which` index (include/p2pvg_b200.h).
    R = 256: 0 / 1 forward MT = 1 / 2, 2 / 3 backward MT = 1 / 2.  R = 512: 0 / 1 / 3 forward MT = 1 / 2 / 3, 2 backward.
    R = 64 and 128 have no diagnostic: {}."""
    if R == 256:
        return {w: int(lib.p2pvg_lstm_cluster_max_clusters(w)) for w in range(4)}
    if R == 512:
        return {w: int(lib.p2pvg_lstm_cluster512_max_clusters(w)) for w in range(4)}
    return {}


def fwd_slab_tiles(B, maxc1):
    """lstm_cluster512.cu:478-492: the MT with the smallest waves * (1.5 + 2.8 MT), in float32, the first one on a tie;
    maxc is the resident-cluster count of the 32-row instance (which = 1), 7 if the query failed."""
    if maxc1 <= 0:
        maxc1 = 7
    best, best_cost = 1, np.float32(0)
    for mt in (1, 2, 3):
        waves = cdiv(cdiv(B, 16 * mt), maxc1)
        cost = np.float32(waves) * (np.float32(1.5) + np.float32(2.8) * np.float32(mt))
        if mt == 1 or cost < best_cost:
            best, best_cost = mt, cost
    return best


@dataclass
class ScanSchedule:
    family: str          # cluster8 | cluster16 | coop-tf32 | coop-exact
    R: int
    B: int
    bwd: bool
    MT: int              # m16 tiles per slab (cooperative: 4, the 64-row block)
    rows: int            # batch rows per slab
    slabs: int
    cs: int              # CTAs per slab (cluster size; cooperative: R/8 CTAs of one row block)
    maxc: object         # resident clusters of this instance, None where no diagnostic exists
    waves: object
    last_rows: int       # valid rows of the last slab
    tf32: bool
    fast_act: bool       # __expf / __fdividef / tanh.approx (cluster kernels) rather than expf / tanhf (cooperative)

    @property
    def units(self):     # hidden units per CTA
        return self.R // self.cs

    def where(self, row, unit):
        slab = row // self.rows
        wave = slab // self.maxc if self.maxc else "?"
        return f"slab {slab} (of {self.slabs}, row {row % self.rows} of it), cluster rank {unit // self.units}, wave {wave}"

    def describe(self):
        d = "bwd" if self.bwd else "fwd"
        return (f"{self.family} {d} R={self.R} B={self.B} MT={self.MT}: {self.slabs} slabs of {self.rows} rows x {self.cs} CTAs, "
                f"max resident {self.maxc}, waves {self.waves}, last slab {self.last_rows} rows")


def scan_schedule(R, B, tf32, maxc, bwd=False):
    """What p2pvg_lstm_scan_fwd (bwd=False) / _bwd launches for (R, B, tf32).  `maxc`: max_clusters(lib, R)."""
    maxc = maxc or {}
    if tf32 and R == 512:                                    # lstm_scan.cu:332 / :340
        if bwd:                                              # lstm_cluster512.cu:504-510: 16-row slabs only
            MT, which = 1, 2
        else:
            MT = fwd_slab_tiles(B, maxc.get(1, 0))           # lstm_cluster512.cu:498
            which = {1: 0, 2: 1, 3: 3}[MT]
        fam, cs, rows = "cluster16", 16, 16 * MT
    elif tf32 and R in (64, 128, 256):                       # lstm_scan.cu:333 / :341; lstm_cluster.cu:367
        MT = 2 if B > MT2_ABOVE else 1                       # lstm_cluster.cu:403 / :416
        which = (2 if bwd else 0) + MT - 1
        fam, cs, rows = "cluster8", 8, 16 * MT
    else:                                                    # lstm_scan.cu:334 / :342, the cooperative scans
        assert R % (64 if bwd else 8) == 0, f"R={R} is not supported by the cooperative scan"
        fam = "coop-tf32" if tf32 else "coop-exact"
        MT, cs, rows, which = COOP_ROWS // 16, R // COOP_UNITS, COOP_ROWS, None
    slabs = cdiv(B, rows)
    if fam.startswith("coop"):
        mc, waves = slabs, 1     # cudaLaunchCooperativeKernel: every CTA is resident, or the launch fails
    else:
        mc = maxc.get(which)
        waves = cdiv(slabs, mc) if mc else None
    return ScanSchedule(fam, R, B, bwd, MT, rows, slabs, cs, mc, waves, B - (slabs - 1) * rows, tf32, fam.startswith("cluster"))


# ------------------------------------------------------------------ operands

def tf32_rna(x):
    """cvt.rna.tf32.f32 on the fp32 bit pattern: round the 13 dropped mantissa bits to nearest, ties away from zero (add half
    of their range, 0x1000, to the magnitude bits), then clear them (mask 0xFFFFE000).  Exact for every finite input whose
    rounded magnitude stays finite."""
    b = x.detach().float().contiguous().view(torch.int32)
    return ((b + 0x1000) & -0x2000).view(torch.float32)


def _operand(x, sched):
    return (tf32_rna(x) if sched.tf32 else x.float()).double()


# ------------------------------------------------------------------ bound constants

U = 2.0 ** -24           # unit roundoff of fp32 round-to-nearest
ULP = 2.0 ** -23         # one ulp relative to a normal fp32 value y is at most 2^-23 |y|
TINY = 2.0 ** -126       # absolute floor: subnormal results, and __fdividef's 0 for a denominator above 2^126 (sigmoid < 2^-126)
# tanh.approx.f32: the PTX ISA gives 2^-10.987 as its maximum error over the whole range.  It is applied as an absolute error;
# |tanh| <= 1, so the bound also holds if the figure is read as relative.
TANH_APPROX = 2.0 ** -10.987


def gamma(n):
    """Higham's gamma_n = n u / (1 - n u): the relative bound of n fp32 roundings (a chain of n fmaf / adds / products)."""
    return n * U / (1 - n * U)


def acc_alpha(sched):
    """Relative bound, to sum |a b| + |other addends|, of the kernel's fp32 sum for one gate pre-activation (forward: K = R)
    or one dh (backward: K = 4R).
    TF32 families: products of tf32 operands are exact in fp32; a chain of m16n8k8 MMAs adds one fp32 accumulation per k8 step
    plus the adds inside one MMA, each off by at most 2^-23 of a partial sum no larger than the magnitude: (K/8 + 16) 2^-23.
    The 16 also covers the few adds after the chain (K-half or partial-product sums, pre + b_hh, dhtop).
    Exact family (lstm_scan.cu): forward, one fmaf chain of R terms then + pre + b_hh (R + 2 roundings); backward, per 256-column
    chunk two chains of 128 fmaf and their sum, one add per chunk into rec, and + dhtop (128 + 1 + 4R/256 + 1)."""
    R = sched.R
    K = 4 * R if sched.bwd else R
    if sched.tf32:
        return (K / 8 + 16) * ULP
    n = (128 + 1 + cdiv(4 * R, 256) + 1) if sched.bwd else R + 2
    return gamma(n)


def sigmoid_err(z, delta, fast):
    """Absolute error of the kernel's sigmoid at an argument within `delta` of z (first-order, with sigma and 1 - sigma at the
    kernel's argument bounded by e^delta times their value at z).
    fast: 1 / (1 + __expf(-x)) by __fdividef.  CUDA C Programming Guide, intrinsic functions: __expf is off by at most
          2 + floor(|1.173 x|) ulp, __fdividef by 2 ulp for denominators in [2^-126, 2^126]; 1 + e rounds once (u).  A relative
          error eps of e moves sigma by (1 - sigma) eps relatively.
    exact: 1.f / (1.f + expf(-x)) (common.cuh:115).  CUDA Math API: expf 2 ulp; the division is IEEE (u), 1 + e rounds (u)."""
    s = torch.sigmoid(z)
    grow = math.exp(delta) if isinstance(delta, float) else torch.exp(delta)
    if fast:
        ne = 2 + torch.floor(1.173 * (z.abs() + delta))
        rel = (1 - s) * grow * ne * ULP + U + 2 * ULP
    else:
        rel = (1 - s) * grow * 2 * ULP + 2 * U
    return s * grow * rel + TINY


def tanh_err(z, delta, fast):
    """Absolute error of the kernel's tanh at an argument within `delta` of z.  fast: tanh.approx.f32 (TANH_APPROX).
    exact: tanhf, 2 ulp (CUDA Math API)."""
    if fast:
        return torch.full_like(z, TANH_APPROX)
    return 2 * ULP * (torch.tanh(z).abs() + delta) + 2.0 ** -148


def gate_bounds(z, delta, R, fast):
    """Reference activations act(z) of [.., 4R] pre-activations (i, f, g, o) and the bound on the kernel's value: the kernel's
    argument is within delta of z, which moves the result by at most act'(z) e^{c delta} delta (|d log sigma'| <= 1,
    |d log tanh'| <= 2), plus the activation's own error."""
    zi, zf, zg, zo = z.split(R, -1)
    di, df, dg, do = delta.split(R, -1)
    refs, bounds = [], []
    for zz, dd, is_tanh in ((zi, di, False), (zf, df, False), (zg, dg, True), (zo, do, False)):
        if is_tanh:
            a = torch.tanh(zz)
            b = (1 - a * a) * torch.exp(2 * dd) * dd + tanh_err(zz, dd, fast)
        else:
            a = torch.sigmoid(zz)
            b = a * (1 - a) * torch.exp(dd) * dd + sigmoid_err(zz, dd, fast)
        refs.append(a)
        bounds.append(b)
    return torch.cat(refs, -1), torch.cat(bounds, -1)


# ------------------------------------------------------------------ the check

def assert_bound(name, got, ref, bound, sched, s0=0, worst=None):
    """|got - ref| <= bound elementwise over [steps, B, 4R] or [steps, B, R] (step s0 first).  NaN or Inf in `got` fails.  On
    failure: the worst element by step, row, unit and gate, with its slab, cluster rank and wave.  Returns the worst ratio
    (folded into worst[name] if a dict is given)."""
    diff = (got.double() - ref).abs()
    ratio = torch.where(bound > 0, diff / bound.clamp_min(1e-300), torch.where(diff > 0, torch.inf, 0.0))
    ratio = torch.nan_to_num(ratio, nan=torch.inf)
    w = ratio.max().item()
    if w > 1.0:
        s, b, col = (int(i) for i in torch.unravel_index(ratio.argmax(), ratio.shape))
        R = sched.R
        gate, unit = ("ifgo"[col // R], col % R) if got.shape[-1] == 4 * R else ("-", col)
        bad = int((ratio > 1.0).sum().item())
        raise AssertionError(
            f"{name} ({sched.describe()}): {bad}/{ratio.numel()} elements out of bound, worst ratio {w:.3g} at step {s0 + s}, "
            f"row {b}, unit {unit}, gate {gate}: got {got[s, b, col].item():.7g}, ref {ref[s, b, col].item():.7g}, "
            f"bound {bound[s, b, col].item():.3g}; {sched.where(b, unit)}")
    if worst is not None:
        worst[name] = max(worst.get(name, 0.0), w)
    return w


def report(worst, sched):
    print(f"[schedule] {sched.describe()}")
    for k, v in worst.items():
        print(f"[bound] {k}: worst error/bound {v:.3g}")


def check_forward(sched, pre, whh, bhh, gates, hs, cs, worst=None, max_elems=1 << 23):
    """Teacher-forced forward check, vectorised over steps (in chunks of at most max_elems float64 per [.., 4R] tensor):
      gates_s vs act(z), z = pre_s + b_hh + rho(hs[s]) rho(W_hh)^T, |delta z| <= acc_alpha * (|pre| + |b| + |rho h| |rho W|^T)
      cs[s+1] vs f gates_s c[s] + i g from the kernel's own gates and c (two roundings: gamma_2)
      hs[s+1] vs o tanh(cs[s+1])                                      (tanh error + one product rounding)"""
    worst = {} if worst is None else worst
    S, B, R4 = gates.shape
    R = R4 // 4
    W = _operand(whh, sched)
    Wa = W.abs()
    b = bhh.double()
    alpha = acc_alpha(sched)
    fast = sched.fast_act
    chunk = max(1, max_elems // (B * R4))
    for s0 in range(0, S, chunk):
        s1 = min(S, s0 + chunk)
        h = _operand(hs[s0:s1], sched)
        p = pre[s0:s1].double()
        z = p + b + h @ W.t()
        delta = alpha * (p.abs() + b.abs() + h.abs() @ Wa.t())
        del h, p
        ref, bound = gate_bounds(z, delta, R, fast)
        del z, delta
        assert_bound("gates", gates[s0:s1], ref, bound, sched, s0, worst)
        del ref, bound
        gk = gates[s0:s1].double()
        i, f, g, o = gk.split(R, -1)
        cprev, cnow = cs[s0:s1].double(), cs[s0 + 1:s1 + 1].double()
        fc, ig = f * cprev, i * g
        assert_bound("c", cs[s0 + 1:s1 + 1], fc + ig, gamma(2) * (fc.abs() + ig.abs()) + TINY, sched, s0, worst)
        tc = torch.tanh(cnow)
        te = tanh_err(cnow, 0.0, fast)
        assert_bound("h", hs[s0 + 1:s1 + 1], o * tc, o.abs() * te + U * o.abs() * (tc.abs() + te) + TINY, sched, s0, worst)
    return worst


def check_backward(sched, dhtop, whh, gates, cs, dG, worst=None):
    """Teacher-forced backward check, step by step from s = S-1 down:
      dh_s = dhtop_s + rho(dG[s+1]) rho(W_hh)   (dhtop alone at s = S-1), |error| <= e_dh = acc_alpha * (|dhtop| + |rho dG| |rho W|)
      dc_s = dh_s o_s (1 - tanh^2 c_s) + f_{s+1} dc_{s+1}, carried in float64 from the kernel's gates and cs, with its error bound
      E_s = e_s + f_{s+1} E_{s+1}; e_s holds the dh error, the tanh error and the fp32 roundings of the dc expression.
    All four gate gradients of every step are compared."""
    worst = {} if worst is None else worst
    S, B, R4 = gates.shape
    R = R4 // 4
    W = _operand(whh, sched)
    Wa = W.abs()
    alpha = acc_alpha(sched)
    fast = sched.fast_act
    dc = torch.zeros(B, R, dtype=torch.float64, device=gates.device)
    E = torch.zeros_like(dc)
    fnext = torch.zeros_like(dc)
    for s in range(S - 1, -1, -1):
        dht = dhtop[s].double()
        if s == S - 1:
            dh, edh = dht, torch.zeros_like(dht)
        else:
            gn = _operand(dG[s + 1], sched)
            dh = dht + gn @ W
            edh = alpha * (dht.abs() + gn.abs() @ Wa)
        i, f, g, o = gates[s].double().split(R, -1)
        cprev, c = cs[s].double(), cs[s + 1].double()
        tc = torch.tanh(c)
        T = tanh_err(c, 0.0, fast)
        D1 = 2 * tc.abs() * T + T * T                       # |(1 - tc_k^2) - (1 - tc^2)|
        one_t = 1 - tc * tc
        dcn = dh * o * one_t + fnext * dc
        e = (o.abs() * (one_t.abs() + D1) * edh + dh.abs() * o.abs() * D1
             + gamma(5) * ((dh.abs() + edh) * o.abs() * (1 + tc * tc + D1) + fnext.abs() * (dc.abs() + E)))
        E = e + fnext.abs() * E
        dc = dcn
        dca = dc.abs() + E
        oo = o * (1 - o)
        ref = torch.cat([dc * g * i * (1 - i), dc * cprev * f * (1 - f), dc * i * (1 - g * g), dh * tc * oo], -1)
        bound = torch.cat([
            (g * i * (1 - i)).abs() * E + gamma(4) * dca * (g * i * (1 - i)).abs(),
            (cprev * f * (1 - f)).abs() * E + gamma(4) * dca * (cprev * f * (1 - f)).abs(),
            (i * (1 - g * g)).abs() * E + gamma(4) * dca * i.abs() * ((1 - g * g).abs() + g * g),
            (tc * oo).abs() * edh + dh.abs() * oo.abs() * T + gamma(4) * (dh.abs() + edh) * (tc.abs() + T) * oo.abs(),
        ], -1) + TINY
        assert_bound("dG", dG[s:s + 1], ref.unsqueeze(0), bound.unsqueeze(0), sched, s, worst)
        fnext = f
    return worst
