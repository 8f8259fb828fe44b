"""Edge cases of the generic kernel's STDP update (``phase3``, csrc/snn_phases.cuh) and of the single-operator kernels
(csrc/snn_ops.cu), with plain float64 restatements of the reference's formulas.  Shared by tests/test_kernel_edges.py
(CPU: the oracle against float64, the emulated kernel against the oracle) and tests/test_gpu_kernel_edges.py (the CUDA
library).  No test functions here.

The cases straddle the thresholds where phase3 changes path:

* target traces staged in shared memory while 32 * 4 * B <= SNN_XT_MAX_BYTES (B <= 768), else read per sample;
* eager weight-row prefetch for B >= 64;
* the first SNN_P3_MAXEV = 16 samples with a post-synaptic event in a 32-column tile get a staging slot, the others
  read the pre-synaptic trace from global memory;
* untouched rows skipped when the pass is not a full one (t > 0 of a window, no decay);
* 32-column tiles and 32-row groups with tails (n not a multiple of 32);

and where the single operators do: ``conn_compute_kernel`` loops over the batch once B > 64 * 8 = 512,
``normalize_tile`` splits the rows into 16 chunks (empty ones for n_src < 16), a zero column takes the ``tot == 0 -> 1``
guard.

Error bound
-----------
With u = 2**-24 (fp32 unit roundoff) and gamma_k = k u / (1 - k u), a value computed from exact inputs by a chain of k
roundings (+, -, *, / in any order) is the exact value times (1 + theta_k), |theta_k| <= gamma_k (Higham, *Accuracy and
Stability of Numerical Algorithms*, Lemma 3.1).  A sum of products evaluated in fp32 in any order, where each term
passes through at most k roundings, therefore differs from its exact (float64) value by at most gamma_k times the sum of
the absolute values of its terms (ibid. §3.1, the same argument as for inner products).

One update of PostPre (reference learning.py:390-420 and :87-104) computes per synapse

    w' = clamp(((w - reduce_b s_b x_b nu0 [* dt]) + reduce_b x_b s_b nu1 [* dt]) * decay)

Term by term: ``x * nu0`` is one rounding, ``s * (x nu0)`` is exact (s in {0, 1}), the batch sum passes a term through
at most B additions, the mean one division, MCC's ``* dt`` one product, the pre and post subtractions two, the decay one:
at most B + 6 roundings, so

    |w'_fp32 - w'_f64| <= gamma_{B+8} * (|w| + sum_b |nu0 s x| + sum_b |nu1 x s|)     (mean: both sums / B)

The clamp is 1-Lipschitz and adds nothing.  WeightDependentPostPre (:626-653) multiplies the reduced sums by nu and by
(w - wmin) resp. (wmax - w) (three roundings per factor chain) and accumulates ``upd`` (two more): its terms are
|nu0| sum_b |s x| |w - wmin| and |nu1| sum_b |x s| |wmax - w|, still within B + 8 roundings.  Hebbian (:1110-1136) is
PostPre with the nu applied after the reduction.  ``gamma_{B+8}`` covers all of them; the two spare roundings make the
constant independent of the rule.

Over a window of T steps the traces are products of up to T decays (nodes.py:96-103), each one rounding, so a trace
carries theta_T and every term of a step gains T roundings: gamma_{B+T+8}.  An error already in w is carried into the
next step with a factor of magnitude <= 1 (1 for PostPre and Hebbian, |1 - nu0 U - nu1 V| for the weight-dependent
form with nu0 U, nu1 V in [0, 1], ``decay`` <= 1, the clamp), so the window's bound is the sum of the per-step bounds,
each taken with |w| widened by the error bound so far.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import torch

U32 = 2.0 ** -24
P3_MAXEV = 16          # SNN_P3_MAXEV (snn_phases.cuh)
XT_STAGED_MAX_B = 768  # phase3 stages the target traces while 32 * 4 * B <= SNN_XT_MAX_BYTES
EAGER_B = 64           # phase3 prefetches weight rows for B >= 64


def gamma(k: int) -> float:
    return k * U32 / (1.0 - k * U32)


def f32(v: float) -> float:
    """``v`` as the fp32 value the kernels hold (the reference's nu is a float32 tensor)."""
    return float(np.float32(v))


# ---- single-operator update cases (snn_b200_conn_update, every rule.update()) -----------------------------------------

RULES = ("postpre", "wdep", "hebbian", "mcc", "noop")
PATTERNS = ("silent", "sparse", "allcols", "single", "deadrows", "zeros")


@dataclass(frozen=True)
class UpdateCase:
    rule: str            # one of RULES; "mcc" is MCC_learning.PostPre on a MulticompartmentConnection with dt = 0.5
    red: str             # "sum", "mean" or "squeeze" (B = 1, reduction left to the rule's default)
    B: int
    ns: int
    nt: int
    pattern: str         # one of PATTERNS
    decay: bool = False  # weight decay 0.0625 (factor 0.9375, exact in fp32)
    bounds: str = "finite"   # "finite" or "inf"
    nu_off: int = -1     # 0: nu0 = 0, 1: nu1 = 0, -1: both on
    recurrent: bool = False  # source is target (ns == nt)
    seed: int = 0

    @property
    def name(self) -> str:
        extra = "".join([f"_nu{self.nu_off}off" if self.nu_off >= 0 else "", "_decay" if self.decay else "",
                         "_inf" if self.bounds == "inf" else "", "_rec" if self.recurrent else "",
                         f"_s{self.seed}" if self.seed else ""])
        return f"b{self.B}_{self.rule}_{self.red}_{self.pattern}_{self.ns}x{self.nt}{extra}"

    @property
    def pre_on(self) -> bool:
        return self.rule != "noop" and self.nu_off != 0

    @property
    def post_on(self) -> bool:
        return self.rule != "noop" and self.nu_off != 1

    @property
    def overflow(self) -> bool:
        """More than P3_MAXEV samples have a post-synaptic event in one tile (the slot-less fallback runs)."""
        return self.pattern == "allcols" and self.B > P3_MAXEV and self.post_on

    @property
    def unstaged(self) -> bool:
        """The target traces are read per sample instead of being staged in shared memory."""
        return self.B > XT_STAGED_MAX_B and self.pre_on


def _validate(c: UpdateCase) -> UpdateCase:
    assert c.rule in RULES and c.pattern in PATTERNS and c.red in ("sum", "mean", "squeeze"), c
    assert (c.red == "squeeze") == (c.B == 1) or c.red != "squeeze", c
    assert not c.recurrent or c.ns == c.nt, c
    assert c.rule != "wdep" or c.bounds == "finite", "WeightDependentPostPre needs finite bounds"
    assert c.rule != "noop" or c.decay, "NoOp without decay changes nothing"
    assert not (c.rule == "mcc" and c.recurrent), c
    return c


def _fixed_update_cases():
    C = UpdateCase
    cases = [
        # B = 1: the squeeze reduction, single columns and rows, word tails
        C("postpre", "squeeze", 1, 784, 1, "sparse"),
        C("wdep", "squeeze", 1, 1, 95, "single"),
        C("mcc", "squeeze", 1, 33, 31, "sparse", decay=True),
        C("hebbian", "sum", 1, 32, 33, "zeros", bounds="inf"),
        C("postpre", "sum", 2, 31, 32, "single", nu_off=0),
        C("postpre", "sum", 2, 33, 33, "silent", recurrent=True),
        # the 16 event slots of a tile: 16 samples fit, 17 and more take the slot-less fallback
        C("postpre", "sum", 16, 33, 95, "allcols"),
        C("postpre", "sum", 17, 33, 95, "allcols"),
        C("wdep", "sum", 17, 257, 31, "allcols"),
        C("postpre", "mean", 31, 31, 31, "allcols", recurrent=True),
        C("hebbian", "sum", 32, 32, 33, "allcols", decay=True),
        C("mcc", "mean", 33, 257, 95, "allcols"),
        C("postpre", "sum", 33, 31, 1, "allcols", nu_off=0),
        # eager weight-row prefetch from B = 64
        C("postpre", "sum", 63, 784, 33, "sparse"),
        C("postpre", "sum", 64, 784, 33, "sparse"),
        C("wdep", "sum", 64, 257, 95, "zeros"),
        C("wdep", "mean", 65, 784, 32, "deadrows"),
        C("hebbian", "sum", 63, 33, 95, "single", bounds="inf"),
        C("postpre", "sum", 65, 257, 1, "allcols", bounds="inf"),
        C("noop", "sum", 64, 31, 95, "sparse", decay=True),
        C("postpre", "sum", 129, 257, 95, "single", nu_off=1),
        C("mcc", "sum", 129, 784, 95, "deadrows", bounds="inf"),
        C("postpre", "sum", 129, 32, 32, "deadrows", recurrent=True, bounds="inf"),
        # staged target traces up to B = 768, per-sample reads from 769
        C("postpre", "sum", 768, 257, 95, "deadrows"),
        C("postpre", "sum", 769, 257, 95, "deadrows"),
        C("postpre", "mean", 768, 33, 33, "allcols"),
        C("postpre", "mean", 769, 33, 33, "allcols"),
        C("wdep", "sum", 769, 784, 31, "sparse", decay=True),
        C("hebbian", "mean", 769, 257, 32, "zeros", decay=True),
        C("mcc", "sum", 1024, 257, 95, "deadrows", decay=True),
        C("postpre", "sum", 1024, 784, 95, "allcols"),
        C("postpre", "sum", 1024, 33, 33, "single", recurrent=True),
        C("wdep", "mean", 1024, 31, 95, "silent"),
        C("hebbian", "sum", 1024, 257, 33, "sparse", nu_off=1, bounds="inf"),
        C("noop", "sum", 1024, 257, 95, "sparse", decay=True),
        C("postpre", "sum", 1024, 1, 95, "deadrows", nu_off=1),
    ]
    return [_validate(c) for c in cases]


def _random_update_cases(count: int = 40, seed: int = 20261015):
    g = np.random.default_rng(seed)
    Bs = (1, 2, 16, 17, 31, 32, 33, 63, 64, 65, 129, 768, 769, 1024)
    out = []
    while len(out) < count:
        rule = RULES[g.integers(len(RULES))]
        B = int(Bs[g.integers(len(Bs))])
        red = "squeeze" if B == 1 and g.random() < 0.5 else ("mean" if g.random() < 0.3 else "sum")
        recurrent = rule != "mcc" and g.random() < 0.2
        ns = int((1, 31, 32, 33, 257, 784)[g.integers(6)])
        nt = int((1, 31, 32, 33, 95)[g.integers(5)])
        if recurrent:
            ns = nt = int((31, 32, 33)[g.integers(3)])
        c = UpdateCase(rule, red, B, ns, nt, PATTERNS[g.integers(len(PATTERNS))],
                       decay=rule == "noop" or bool(g.random() < 0.3),
                       bounds="finite" if rule == "wdep" or g.random() < 0.6 else "inf",
                       nu_off=int(g.choice([-1, -1, -1, 0, 1])) if rule != "noop" else -1,
                       recurrent=recurrent, seed=len(out) + 1)
        out.append(_validate(c))
    return out


UPDATE_CASES = _fixed_update_cases() + _random_update_cases()


def draw_update(c: UpdateCase) -> dict:
    """The seeded spikes, traces and weights of a case, on the CPU, float32 / bool."""
    g = torch.Generator().manual_seed(7919 * c.seed + 31 * c.B + 7 * c.ns + c.nt)
    B, ns, nt = c.B, c.ns, c.nt

    def traces(n):
        x = torch.rand(B, n, generator=g)
        return torch.where(torch.rand(B, n, generator=g) < 0.2, torch.zeros(()), x)   # exact zeros among them

    x_src, x_tgt = traces(ns), traces(nt)
    s_src = torch.rand(B, ns, generator=g) < 0.25
    s_tgt = torch.zeros(B, nt, dtype=torch.bool)
    if c.pattern == "silent":
        s_src[:] = False
    elif c.pattern in ("sparse", "zeros"):
        s_tgt = torch.rand(B, nt, generator=g) < 0.05
    elif c.pattern == "allcols":   # every sample spikes in the same columns: all samples have an event in their tiles
        for j in sorted({0, nt // 2, nt - 1, min(nt - 1, 40)}):
            s_tgt[:, j] = True
    elif c.pattern == "single":    # one sample has post-synaptic events, nobody else
        b = (B * 2) // 3
        s_tgt[b] = torch.rand(nt, generator=g) < 0.3
        s_tgt[b, nt - 1] = True
    elif c.pattern == "deadrows":  # most samples' target-trace rows are all zero: the live-sample skip
        dead = torch.rand(B, generator=g) < 0.85
        dead[B // 2] = False
        x_tgt[dead] = 0.0
        s_tgt = torch.rand(B, nt, generator=g) < 0.03
    if c.recurrent:   # one layer: its spikes and traces are both ends of the update
        s_src = s_tgt = s_src | s_tgt
        x_src = x_tgt
    if c.bounds == "finite":
        wmin, wmax = (-1.0, 1.0) if c.rule in ("hebbian", "noop") else (0.0, 1.0)
        w = wmin + (wmax - wmin) * (0.1 + 0.8 * torch.rand(ns, nt, generator=g))
    else:
        wmin, wmax = -np.inf, np.inf
        w = 2.0 * torch.rand(ns, nt, generator=g) - 0.5
    if c.pattern == "zeros":      # exact zeros (and negative zeros) among the weights
        z = torch.rand(ns, nt, generator=g)
        w = torch.where(z < 0.3, torch.zeros(()), w)
        w = torch.where(z < 0.1, torch.full((), -0.0), w)
    # nu scaled with 1/B (sum) so that a large batch moves the weights about as far as a small one, without saturating
    scale = 1.0 if c.red == "mean" else 1.0 / B
    nu0, nu1 = f32(0.35 * scale), f32(0.6 * scale)
    if c.rule == "mcc":
        nu0, nu1 = f32(0.5 * nu0), f32(0.5 * nu1)
    if c.nu_off == 0:
        nu0 = 0.0
    if c.nu_off == 1:
        nu1 = 0.0
    return dict(w=w.contiguous(), s_src=s_src.contiguous(), x_src=x_src.contiguous(), s_tgt=s_tgt.contiguous(),
                x_tgt=x_tgt.contiguous(), nu0=nu0, nu1=nu1, wmin=wmin, wmax=wmax,
                wd=0.0625 if c.decay else 0.0, dt=0.5 if c.rule == "mcc" else 1.0)


def build_update(ns, c: UpdateCase, d: dict):
    """The connection of a case with its layers' s / x set (CPU tensors).  Returns (conn, source, target)."""
    N, T = ns.nodes, ns.topology
    B = c.B
    if c.recurrent:
        X = Y = N.LIFNodes(c.nt, traces=True)
    else:
        X, Y = N.Input(c.ns, traces=True), N.LIFNodes(c.nt, traces=True)
    for l in {id(X): X, id(Y): Y}.values():
        l.compute_decays(1.0)
        l.set_batch_size(B)
    X.s, X.x = d["s_src"].clone(), d["x_src"].clone()
    if not c.recurrent:
        Y.s, Y.x = d["s_tgt"].clone(), d["x_tgt"].clone()
    red = {"sum": torch.sum, "mean": torch.mean, "squeeze": None}[c.red]
    if c.rule == "mcc":
        from bindsnet_b200.learning.MCC_learning import PostPre as MccPostPre
        from bindsnet_b200.network.topology_features import Weight

        feat = Weight("weight", d["w"].clone(), range=[d["wmin"], d["wmax"]], learning_rule=MccPostPre,
                      nu=[d["nu0"], d["nu1"]], reduction=red, decay=d["wd"])
        conn = T.MulticompartmentConnection(X, Y, pipeline=[feat])
        conn.dt = d["dt"]
        return conn, X, Y
    L = ns.learning
    rule = {"postpre": L.PostPre, "wdep": L.WeightDependentPostPre, "hebbian": L.Hebbian, "noop": L.NoOp}[c.rule]
    conn = T.Connection(X, Y, w=d["w"].clone(), update_rule=rule, nu=(d["nu0"], d["nu1"]), reduction=red,
                        weight_decay=d["wd"], wmin=d["wmin"], wmax=d["wmax"])
    return conn, X, Y


def run_update(ns, c: UpdateCase, d: dict, device: str = "cpu") -> torch.Tensor:
    """``conn.update(learning=True)`` once; returns the weights after it (CPU).  On the CPU the caller routes the
    single operators to the oracle or the emulated kernel."""
    conn, X, Y = build_update(ns, c, d)
    if device != "cpu":
        for m in {id(X): X, id(Y): Y, id(conn): conn}.values():
            m.to(device)
    conn.update(learning=True)
    return conn.w.detach().cpu().clone()


def ref_update(c: UpdateCase, d: dict):
    """One update in float64, restating the reference: PostPre learning.py:390-420, WeightDependentPostPre :626-653,
    Hebbian :1110-1136, MCC_learning.PostPre MCC_learning.py:224-302, then the base class (learning.py:87-104,
    MCC_learning.py:86-110): pre term, post term, decay, clamp.  Batch reductions are matrix products.
    Returns (w, bound) — the error bound of the module docstring."""
    f = torch.float64
    w = d["w"].to(f)
    sS, xS, sT, xT = (d[k].to(f) for k in ("s_src", "x_src", "s_tgt", "x_tgt"))
    w, bound = _rule_step(c.rule, c.red == "mean", w, sS, xS, sT, xT, d, gamma(c.B + 8), torch.zeros_like(w))
    return w, bound


def _rule_step(rule, mean, w, sS, xS, sT, xT, d, gam, err):
    """One application of the rule in float64; ``err`` is the error bound w carries in.  Returns (w', bound')."""
    B = sS.shape[0]
    nu0, nu1, wmin, wmax, dt = d["nu0"], d["nu1"], d["wmin"], d["wmax"], d["dt"]
    red = (lambda m: m / B) if mean else (lambda m: m)
    terms = w.abs() + err
    w0 = w
    if rule in ("postpre", "mcc"):
        scale = dt if rule == "mcc" else 1.0
        if nu0 != 0.0:   # learning.py:399-405 / MCC_learning.py:233-263
            w = w - red(sS.T @ (xT * nu0)) * scale
            terms = terms + red(sS.T @ (xT * nu0).abs()) * scale
        if nu1 != 0.0:   # learning.py:409-417 / MCC_learning.py:267-299
            w = w + red(xS.T @ (sT * nu1)) * scale
            terms = terms + red(xS.abs().T @ (sT * nu1).abs()) * scale
    elif rule == "wdep":   # learning.py:639-651
        upd = torch.zeros_like(w)
        if nu0 != 0.0:
            P = red(sS.T @ xT)
            upd = upd - nu0 * P * (w0 - wmin)
            terms = terms + abs(nu0) * red(sS.T @ xT.abs()) * ((w0 - wmin).abs() + err)
        if nu1 != 0.0:
            Q = red(xS.T @ sT)
            upd = upd + nu1 * Q * (wmax - w0)
            terms = terms + abs(nu1) * red(xS.abs().T @ sT) * ((wmax - w0).abs() + err)
        w = w + upd
    elif rule == "hebbian":   # learning.py:1123-1133
        w = w + nu0 * red(sS.T @ xT)
        w = w + nu1 * red(xS.T @ sT)
        terms = terms + abs(nu0) * red(sS.T @ xT.abs()) + abs(nu1) * red(xS.abs().T @ sT)
    factor = 1.0 - d["wd"] if d["wd"] else 1.0   # learning.py:85, :93-94
    w = w * factor
    if rule != "noop" and (wmin != -np.inf or wmax != np.inf):   # learning.py:97-104
        w = w.clamp(wmin, wmax)
    return w, err + gam * terms


def tile_event_counts(s_tgt: torch.Tensor) -> int:
    """The largest number of samples with a post-synaptic event in one 32-column tile."""
    B, nt = s_tgt.shape
    pad = torch.zeros(B, (nt + 31) // 32 * 32, dtype=torch.bool)
    pad[:, :nt] = s_tgt
    return int(pad.view(B, -1, 32).any(2).sum(0).max())


def check_bites(c: UpdateCase, d: dict, w_after: torch.Tensor, interior_min: float = 0.5):
    """What the case claims to exercise, it does: weights changed (or, silent, did not), the clamp did not decide the
    result, the overflow and unstaged paths are reached."""
    w0 = d["w"]
    changed = w_after.view(torch.int32) != w0.view(torch.int32)
    if c.pattern == "silent" and not c.decay:
        assert not changed.any(), f"{c.name}: a silent step changed {int(changed.sum())} weights"
        return
    assert changed.any(), f"{c.name}: no weight changed"
    if c.bounds == "finite" and c.rule != "noop":
        v = w_after[changed]
        inside = ((v > d["wmin"]) & (v < d["wmax"])).float().mean().item()
        assert inside >= interior_min, f"{c.name}: only {inside:.2f} of the changed weights are inside (wmin, wmax)"
    if c.overflow:
        n = tile_event_counts(d["s_tgt"])
        assert n > P3_MAXEV, f"{c.name}: claims the slot overflow, but at most {n} samples have an event in a tile"
    if c.unstaged:
        assert c.B > XT_STAGED_MAX_B and c.pre_on


def ratio(w: torch.Tensor, w64: torch.Tensor, bound: torch.Tensor) -> float:
    """max |w - w64| / bound; an entry with bound 0 must be exact (ratio inf otherwise)."""
    diff = (w.to(torch.float64) - w64).abs()
    if bool((diff[bound == 0] > 0).any()):
        return float("inf")
    pos = bound > 0
    return float((diff[pos] / bound[pos]).max()) if bool(pos.any()) else 0.0


# ---- window cases: phase3 at t > 0 with a target raster that does not depend on rounding ----------------------------

@dataclass(frozen=True)
class WindowCase:
    B: int
    nt: int
    rule: str = "postpre"    # postpre / wdep / hebbian
    red: str = "sum"
    decay: bool = False
    bounds: str = "finite"
    ns: int = 48             # the CPU emulation's size; the GPU runs n_src = 784
    T: int = 30
    seed: int = 0

    @property
    def name(self) -> str:
        return (f"b{self.B}_{self.rule}_{self.red}_{self.ns}x{self.nt}_T{self.T}" + ("_decay" if self.decay else "") +
                ("_inf" if self.bounds == "inf" else ""))


WINDOW_CASES = [
    WindowCase(1, 33),
    WindowCase(48, 95, "wdep"),
    WindowCase(64, 1, "postpre", "mean"),
    WindowCase(200, 33, "hebbian", bounds="inf"),
    WindowCase(769, 95, "postpre", decay=True),
    WindowCase(1024, 33, "wdep", "mean"),
    WindowCase(1024, 95, "postpre"),
]


def draw_window(c: WindowCase) -> dict:
    g = torch.Generator().manual_seed(104729 + c.B * 131 + c.nt + c.seed)
    T, B, ns, nt = c.T, c.B, c.ns, c.nt
    x_in = (torch.rand(T, B, ns, generator=g) < 0.15).to(torch.uint8)
    z_in = (torch.rand(T, B, nt, generator=g) < torch.linspace(0.02, 0.3, B).view(1, B, 1)).to(torch.uint8)
    if c.bounds == "finite":
        wmin, wmax = (-1.0, 1.0) if c.rule == "hebbian" else (0.0, 1.0)
        w = wmin + (wmax - wmin) * (0.2 + 0.6 * torch.rand(ns, nt, generator=g))
    else:
        wmin, wmax = -np.inf, np.inf
        w = torch.rand(ns, nt, generator=g) - 0.3
    scale = 1.0 if c.red == "mean" else 1.0 / B
    return dict(x_in=x_in, z_in=z_in, w=w.contiguous(), nu0=f32(0.02 * scale), nu1=f32(0.03 * scale), wmin=wmin,
                wmax=wmax, wd=0.0625 if c.decay else 0.0, dt=1.0)


# Y's threshold is so far above rest that the learned input (|w| <= 1 + drift, at most n_src spikes a step, summed over
# the window) cannot reach it; Z's input (Z_GAIN through the identity) always does.  With refrac = 0, Y spikes exactly
# one step after Z does, in every sample — whatever the learned weights round to.
Y_THRESH, Z_GAIN = 1.0e6, 1.0e8


def build_window(ns_, c: WindowCase, d: dict):
    N, T, L = ns_.nodes, ns_.topology, ns_.learning
    net = ns_.Network(dt=1.0, batch_size=c.B, learning=True)
    X, Z = N.Input(c.ns, traces=True), N.Input(c.nt)
    Y = N.LIFNodes(c.nt, traces=True, thresh=Y_THRESH, refrac=0)
    net.add_layer(X, "X"); net.add_layer(Z, "Z"); net.add_layer(Y, "Y")
    rule = {"postpre": L.PostPre, "wdep": L.WeightDependentPostPre, "hebbian": L.Hebbian}[c.rule]
    red = {"sum": torch.sum, "mean": torch.mean}[c.red]
    net.add_connection(T.Connection(X, Y, w=d["w"].clone(), update_rule=rule, nu=(d["nu0"], d["nu1"]), reduction=red,
                                    weight_decay=d["wd"], wmin=d["wmin"], wmax=d["wmax"]), "X", "Y")
    net.add_connection(T.Connection(Z, Y, w=Z_GAIN * torch.eye(c.nt)), "Z", "Y")
    from bindsnet_b200.network.monitors import Monitor

    net.add_monitor(Monitor(Y, ["s"], time=c.T), "Ys")
    return net, {"X": d["x_in"], "Z": d["z_in"]}


def window_state(net) -> dict:
    return {"w": net.connections[("X", "Y")].w.detach().cpu().clone(),
            "Ys": net.monitors["Ys"].get("s").cpu().reshape(net.monitors["Ys"].get("s").shape[0], -1).bool(),
            "Xx": net.layers["X"].x.detach().cpu().clone(), "Yx": net.layers["Y"].x.detach().cpu().clone()}


def ref_window(c: WindowCase, d: dict, trace_decay: float):
    """The window replayed in float64: Y's raster is Z's, one step later (network.py:211-250 feeds the previous step's
    spikes); the traces follow nodes.py:96-103 (decay, then set to 1 on a spike) with the layers' fp32 decay factor; the
    rule as in ``ref_update``.  Returns (w, bound, raster of Y [T, B, nt] bool)."""
    f = torch.float64
    T, B = c.T, c.B
    w, err = d["w"].to(f), torch.zeros(c.ns, c.nt, dtype=f)
    xX, xY = torch.zeros(B, c.ns, dtype=f), torch.zeros(B, c.nt, dtype=f)
    sY = torch.zeros(B, c.nt, dtype=torch.bool)
    ys = []
    gam = gamma(B + T + 8)
    for t in range(T):
        sX = d["x_in"][t].bool()
        sY = d["z_in"][t - 1].bool() if t > 0 else torch.zeros(B, c.nt, dtype=torch.bool)
        xX = torch.where(sX, torch.ones((), dtype=f), xX * trace_decay)
        xY = torch.where(sY, torch.ones((), dtype=f), xY * trace_decay)
        w, err = _rule_step(c.rule, c.red == "mean", w, sX.to(f), xX, sY.to(f), xY, d, gam, err)
        ys.append(sY)
    return w, err, torch.stack(ys)


# ---- single operators: Connection.compute / normalize, the MCC feature normalize, Conv2dConnection -----------------

def compute_setup(ns_, n_src: int, n_tgt: int, B: int, bias: bool, seed: int = 0):
    """A dense Connection and ALL-spiking inputs [B, n_src] (every row of the weights enters every output)."""
    g = torch.Generator().manual_seed(300 + seed + n_src + B)
    X, Y = ns_.nodes.Input(n_src), ns_.nodes.LIFNodes(n_tgt)
    w = torch.rand(n_src, n_tgt, generator=g) - 0.25
    b = torch.rand(n_tgt, generator=g) if bias else None
    conn = ns_.topology.Connection(X, Y, w=w, b=b)
    s = torch.ones(B, n_src, dtype=torch.bool)
    s[B // 3, n_src // 2] = False   # and one silent input, so a spike-gather that ignores s would be caught
    return conn, s


def ref_compute(conn, s):
    """topology.py:332-346: s.float() @ w + b, in float64.  Bound: a sum of n_src + 1 terms in ascending order."""
    w = conn.w.detach().cpu().to(torch.float64)
    sd = s.cpu().to(torch.float64)
    out = sd @ w
    absum = sd @ w.abs()
    if conn.b is not None:
        out = out + conn.b.detach().cpu().to(torch.float64)
        absum = absum + conn.b.detach().cpu().to(torch.float64).abs()
    return out, gamma(w.shape[0] + 1) * absum


def poisoned(w: torch.Tensor, extra_rows: int = 64) -> torch.Tensor:
    """``w`` copied into the head of a larger buffer whose tail is NaN: a kernel that reads rows past n_src (a chunk
    bound without its ``min``) turns its column sums into NaN instead of reading whatever follows the tensor."""
    n, m = w.shape
    buf = torch.full(((n + extra_rows) * m,), float("nan"), dtype=w.dtype, device=w.device)
    out = buf[: n * m].view(n, m)
    out.copy_(w)
    return out


def normalize_setup(ns_, n_src: int, n_tgt: int = 37, mcc: bool = False, seed: int = 0):
    """Connection.normalize (absolute column sums, negative weights) or the MCC Weight feature's normalize (plain
    column sums), with column 3 all zero (the ``tot == 0 -> 1`` guard)."""
    g = torch.Generator().manual_seed(500 + n_src + seed)
    X, Y = ns_.nodes.Input(n_src), ns_.nodes.LIFNodes(n_tgt)
    if mcc:
        from bindsnet_b200.network.topology_features import Weight

        w = torch.rand(n_src, n_tgt, generator=g) + 0.05
        w[:, 3] = 0.0
        return ns_.topology.MulticompartmentConnection(X, Y, pipeline=[Weight("weight", w, norm=7.5)])
    w = torch.rand(n_src, n_tgt, generator=g) - 0.6
    w[:, 3] = 0.0
    return ns_.topology.Connection(X, Y, w=w, norm=11.0)


def poison_weights(conn) -> None:
    """Move the weights of a (Multicompartment)Connection, on their device, into a buffer with a NaN tail."""
    if hasattr(conn, "pipeline"):
        conn.pipeline[0].value.data = poisoned(conn.pipeline[0].value.data)
    else:
        conn.w.data = poisoned(conn.w.data)


def ref_normalize(w0: torch.Tensor, norm: float, absolute: bool):
    """Connection.normalize topology.py:383-392 (absolute) / AbstractFeature.normalize topology_features.py:250-266
    (plain), in float64: w * norm / colsum, a zero column sum replaced by 1.  Bound: the column sum passes a term
    through at most n_src + 16 additions (16 row chunks), then one division and one product — relative to |w norm /
    colsum| for non-negative summands (the absolute form, and the plain form on non-negative weights)."""
    w = w0.to(torch.float64)
    tot = (w.abs() if absolute else w).sum(0, keepdim=True)
    tot = torch.where(tot == 0, torch.ones((), dtype=torch.float64), tot)
    out = w * (norm / tot)
    return out, gamma(w.shape[0] + 18) * out.abs()


CONV_GEOMETRIES = [
    # (cin, H, W, cout, (kh, kw), (sh, sw), (ph, pw), (dh, dw))
    (1, 7, 5, 3, (3, 2), (1, 1), (0, 0), (1, 1)),
    (2, 9, 6, 4, (3, 3), (2, 1), (1, 0), (1, 1)),
    (3, 5, 8, 2, (2, 4), (1, 3), (0, 2), (1, 1)),
    (2, 3, 4, 3, (5, 6), (1, 1), (2, 3), (1, 1)),     # a kernel wider and taller than the unpadded input
    (1, 6, 4, 2, (7, 2), (2, 2), (3, 1), (1, 1)),
    (2, 10, 7, 3, (3, 2), (1, 2), (1, 1), (2, 3)),    # dilated
    (1, 8, 8, 2, (2, 3), (3, 2), (2, 0), (3, 2)),
]


def conv_setup(ns_, geo, seed: int = 0, B: int = 5):
    cin, H, W, cout, k, st, pad, dil = geo
    g = torch.Generator().manual_seed(900 + seed + H * W)
    oh = (H - k[0] + 2 * pad[0]) // st[0] + 1
    ow = (W - k[1] + 2 * pad[1]) // st[1] + 1
    X = ns_.nodes.Input(shape=[cin, H, W])
    Y = ns_.nodes.LIFNodes(shape=[cout, oh, ow])
    w = torch.rand(cout, cin, *k, generator=g) + 0.02   # positive: the filter sums of normalize() do not cancel
    b = torch.rand(cout, generator=g) - 0.5
    conn = ns_.topology.Conv2dConnection(X, Y, kernel_size=k, stride=st, padding=pad, dilation=dil, w=w, b=b, norm=3.0)
    s = torch.rand(B, cin, H, W, generator=g) < 0.5
    s[0] = True
    return conn, s


def ref_conv_compute(conn, s, w0=None):
    """topology.py:799-815: F.conv2d(s.float(), w, b, stride, padding, dilation) in float64.  The target shape follows
    the reference's formula, which ignores the dilation (topology.py:752-772); where it is larger than F.conv2d's output
    the kernel reads the taps that fall outside the input as zeros, so the input is extended by zeros on the bottom and
    right.  Bound: each output sums at most cin * kh * kw taps and the bias.  ``w0``: the weights compute() saw."""
    import torch.nn.functional as F

    w = (conn.w.detach() if w0 is None else w0).cpu().to(torch.float64)
    b = conn.b.detach().cpu().to(torch.float64)
    sd = s.cpu().to(torch.float64)
    oh, ow = conn.target.shape[1], conn.target.shape[2]
    (kh, kw), (sh, sw), (dh, dw) = conn.kernel_size, conn.stride, conn.dilation
    extra_h = max(0, (oh - 1) * sh + (kh - 1) * dh + 1 - (sd.shape[2] + 2 * conn.padding[0]))
    extra_w = max(0, (ow - 1) * sw + (kw - 1) * dw + 1 - (sd.shape[3] + 2 * conn.padding[1]))
    sd = F.pad(sd, (0, extra_w, 0, extra_h))
    kw_ = dict(stride=conn.stride, padding=conn.padding, dilation=conn.dilation)
    out = F.conv2d(sd, w, b, **kw_)[:, :, :oh, :ow]
    absum = F.conv2d(sd, w.abs(), b.abs(), **kw_)[:, :, :oh, :ow]
    K = w.shape[1] * w.shape[2] * w.shape[3]
    return out, gamma(K + 1) * absum


def ref_conv_normalize(w0: torch.Tensor, norm: float):
    """Conv2dConnection.normalize topology.py:824-837: every (out, in) filter scaled to sum ``norm`` (no zero guard)."""
    w = w0.to(torch.float64)
    tot = w.sum((2, 3), keepdim=True)
    out = w * (norm / tot)
    return out, gamma(w.shape[2] * w.shape[3] + 2) * out.abs()
