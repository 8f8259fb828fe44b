"""Edge cases of the generic kernel's learning paths that only run inside a window — ``phase3_mstdp_dense`` (MSTDP,
MSTDPET and their MulticompartmentConnection forms), ``phase3_conv`` (MSTDP, PostPre, WeightDependentPostPre and Hebbian
on a Conv2dConnection), ``phase3_local2d`` — and of phase 1's convolutional and LocalConnection2D gathers
(``gather_conv``, ``gather_local2d``), with plain float64 restatements of the reference's formulas and Python mirrors of
the conditions where the kernels change path (csrc/snn_phases.cuh).  Shared by tests/test_learning_edges.py (CPU: the
oracle against float64, the emulated kernel against the oracle) and tests/test_gpu_learning_edges.py (the CUDA library).
No test functions here.

Window cases
------------
The learned connection X -> Y is inserted first, so it is the input phase 1 stages (``gain_first`` cases insert the
gain first, and the learned convolution takes the unstaged path).  Y (LIFNodes) has ``thresh = 1e6`` and
``refrac = 0``: the learned input cannot reach it.  An ``Input`` Z drives Y through a gain connection of weight 1e8
without a rule (a 1x1 Conv2dConnection with weights ``1e8 * eye(cout)`` into the ``[cout, h, w]`` target; a dense
target is shaped [1, 1, nt]), so Y spikes exactly one step after Z, in every sample, whatever the learned weights round
to.  The sources are Bernoulli rasters, different in every sample.

Gather cases
------------
The convolutional or local connection feeds a ``McCullochPitts(thresh=1e9)`` whose voltage is its input: a ``Monitor``
on ``v`` records every step's gather, which is compared with a float64 convolution of the previous step's source spikes.

Error bound
-----------
With u = 2**-24 and gamma_k = k u / (1 - k u), a value computed from exact inputs by a sum of terms, each of which passes
through at most k roundings, differs from its exact value by at most gamma_k times the sum of the absolute values of its
terms (Higham, *Accuracy and Stability of Numerical Algorithms*, Lemma 3.1 and §3.1).  The rule constants (decay factors
``exp(-dt / tc)``, nu, a_plus, a_minus, reward) are the fp32 values the reference holds and are taken as exact inputs.

* A trace ``p <- p * decay + a * s`` costs two roundings per step (learning.py:1564-1567); its terms all have the sign
  of ``a`` (a layer trace, nodes.py:96-103, is a product of decays or 1: one rounding per step), so after t steps
  ``|p_fp32 - p| <= gamma_{2t} |p|``.
* An eligibility term adds the two products ``p_plus s_post + s_pre p_minus`` (the products with spikes are exact): one
  addition.  The convolutional eligibility sums up to L = hout * wout positions per part, then adds the parts: L + 1.
* The batch sum passes a term through at most B additions after the product with the reward; ``mean`` adds one division.
* Then ``nu * upd`` (one product), the add to w (one), the decay (one).  The clamp is 1-Lipschitz and adds nothing.
* MSTDPET (learning.py:2229-2236): the eligibility trace ``et <- et * decay_e + e / tc_e`` costs three roundings per
  step (so 3t + 2t + 1 over t steps, the trace terms included); ``nu * dt * reward`` two, times et and the add two more.

So one step of dense MSTDP changes w by terms that each pass through at most 2T + B + 8 roundings, the convolutional
form 2T + L + B + 8, PostPre / WeightDependentPostPre / Hebbian (layer traces) T + L + B + 8 on a convolution (T + B + 8
on a local connection, which has one position per weight), MSTDPET 5T + 8.  Per step the bound is gamma_k times
(|w| + the error carried in + the sum of the absolute update terms); an error already in w is carried into the next
step with a factor of magnitude <= 1 (the update of MSTDP does not depend on w, WeightDependentPostPre's factor is
|1 - nu0 U - nu1 V| <= 1, decay <= 1, clamp), so over a window the per-step bounds add up as in
``kernel_edges.ref_window``.  An entry whose bound is 0 must be exact.

A gather sums at most K = cin * kh * kw taps and the bias: gamma_{K+1} times the sum of their absolute values
(kernel_edges.ref_conv_compute); a LocalConnection2D adds cin channel sums of K terms each: gamma_{cin (K + 1)}.
"""
from __future__ import annotations

from dataclasses import dataclass, replace

import numpy as np
import torch
import torch.nn.functional as F

import kernel_edges as ke
from kernel_edges import Y_THRESH, Z_GAIN, f32, gamma

# csrc/snn_phases.cuh / snn_common.cuh
CONV_STAGE_WORDS = 4096     # SNN_CONV_STAGE_WORDS
CONV_STAGE_TAPS = 4096      # SNN_CONV_STAGE_TAPS
GEN_THREADS, GEN_WARPS, TILE = 256, 8, 32
ACC_FLOATS = GEN_WARPS * 32 * 32    # the 32 KB accumulator region, in floats
DENSE_STAGE_BYTES = 4 * ACC_FLOATS  # sizeof(float) * SNN_GEN_WARPS * 32 * 32
XT_MAX_BYTES = 96 * 1024    # SNN_XT_MAX_BYTES


def nw(n: int) -> int:
    return (n + 31) // 32


# ---- path mirrors: the C conditions, restated ------------------------------------------------------------------------

@dataclass(frozen=True)
class ConvGeo:
    """A Conv2dConnection: source [cin, hin, win] -> target [cout, hout, wout] (the reference's shape formula)."""
    cin: int
    hin: int
    win: int
    cout: int
    k: tuple
    s: tuple = (1, 1)
    p: tuple = (0, 0)
    d: tuple = (1, 1)

    @property
    def hout(self):
        return int((self.hin - self.k[0] + 2 * self.p[0]) / self.s[0] + 1)

    @property
    def wout(self):
        return int((self.win - self.k[1] + 2 * self.p[1]) / self.s[1] + 1)

    @property
    def L(self):
        return self.hout * self.wout

    @property
    def K(self):
        return self.cin * self.k[0] * self.k[1]

    @property
    def ns(self):
        return self.cin * self.hin * self.win

    @property
    def nt(self):
        return self.cout * self.L

    @property
    def tag(self):
        return (f"c{self.cin}x{self.hin}x{self.win}_o{self.cout}_k{self.k[0]}x{self.k[1]}_s{self.s[0]}x{self.s[1]}"
                f"_p{self.p[0]}x{self.p[1]}" + (f"_d{self.d[0]}x{self.d[1]}" if self.d != (1, 1) else ""))


def conv_mstdp_paths(g: ConvGeo, B: int) -> dict:
    """phase3_conv's MSTDP eligibility walk (snn_phases.cuh): bit rows staged in shared memory, source spikes as a
    decoded list, P- rows staged, output channels per unit, the unit-stride shortcut.  (B does not enter.)"""
    Snw, Gnw = nw(g.ns), nw(g.nt)
    staged = Snw + Gnw <= CONV_STAGE_WORDS
    slist_cap = CONV_STAGE_WORDS - Snw - Gnw - (g.cin + 2) if staged else 0
    listed = staged and g.ns <= 65535 and g.hin <= 256 and g.win <= 256 and slist_cap >= g.ns
    stage_pm = g.L <= ACC_FLOATS
    cpc = min(max(1, GEN_THREADS // g.K), ACC_FLOATS // g.L) if stage_pm else max(1, GEN_THREADS // g.K)
    return dict(staged=staged, listed=listed, stage_pm=stage_pm, cpc=cpc, unit_stride=g.s == (1, 1),
                slist_margin=slist_cap - g.ns, multi_channel=g.cin > 1, shuffle_tail=B > 32 and B % 32 != 0)


def dense_mstdp_staged(B: int, nt: int) -> bool:
    """phase3_mstdp_dense stages the rule state when the target-trace region exists (32 * 4 * B <= SNN_XT_MAX_BYTES)
    and ``32 B + 5 B nt + 16`` bytes fit the accumulator region."""
    return 128 * B <= XT_MAX_BYTES and 32 * B + 5 * B * nt + 16 <= DENSE_STAGE_BYTES


def gather_paths(g: ConvGeo, B: int, local: bool = False) -> dict:
    """phase 1's staging of a convolutional (or, ``local``, LocalConnection2D) input that is the first into its target.
    ``st_bits``: True when staged for every sample chunk size (B * S.nw <= 4096), False when for none (S.nw > 4096),
    None when it depends on the chunk (the GPU's and the emulation's differ: plan_units).  ``st_taps_all`` /
    ``st_taps_some_off``: every 32-neuron tile stages its filter taps / some tile does not.  ``funnel``: the kw taps of
    a filter row are cut out of the bit row (dw == 1, kw <= 32) rather than visited one by one."""
    Snw = nw(g.ns)
    st_bits = True if B * Snw <= CONV_STAGE_WORDS else (False if Snw > CONV_STAGE_WORDS else None)
    n, Lhw = g.nt, g.L
    taps = []
    for tile in range(nw(n)):
        co_base = (tile * TILE) // Lhw
        co_hi = min(n - 1, tile * TILE + TILE - 1) // Lhw
        taps.append(not local and (co_hi - co_base + 1) * g.K <= CONV_STAGE_TAPS)
    return dict(st_bits=st_bits, st_taps_all=all(taps), st_taps_some_off=not all(taps),
                funnel=g.d[1] == 1 and g.k[1] <= 32, kw_over_32=g.k[1] > 32,
                word_straddle=g.win % 32 != 0)


# ---- window cases ------------------------------------------------------------------------------------------------------

DENSE_RULES = ("mstdp", "mstdpet", "mcc_mstdp", "mcc_mstdpet")
CONV_RULES = ("mstdp", "postpre", "wdep", "hebbian")
LOCAL_RULES = ("postpre", "wdep", "hebbian")


@dataclass(frozen=True)
class WinCase:
    kind: str                 # "dense", "conv" or "local"
    rule: str
    B: int
    T: int
    ns: int = 0               # dense: source size
    nt: int = 0               # dense: target size
    geo: ConvGeo = None       # conv: the learned convolution; local: (cin, hin, win), n_filters = cout, k, s
    red: str = "sum"
    reward: float = 0.75
    decay: bool = False
    bounds: str = "finite"
    nu_off: int = -1          # STDP rules: 0: nu0 = 0, 1: nu1 = 0
    gain_first: bool = False  # the gain conv is inserted before the learned one (phase 1 stages the gain conv)
    p_src: float = 0.15
    gpu: tuple = ()           # (B, T) on the GPU where the CPU tier runs a smaller size
    claims: tuple = ()        # (switch, side) pairs of the path mirrors this case is there to reach
    seed: int = 0

    @property
    def name(self) -> str:
        shape = f"{self.ns}x{self.nt}" if self.kind == "dense" else self.geo.tag
        extra = "".join([f"_r{self.reward:g}" if self.reward != 0.75 else "", "_decay" if self.decay else "",
                         "_inf" if self.bounds == "inf" else "", f"_nu{self.nu_off}off" if self.nu_off >= 0 else "",
                         "_gainfirst" if self.gain_first else "", f"_s{self.seed}" if self.seed else ""])
        return f"{self.kind}_{self.rule}_b{self.B}_t{self.T}_{self.red}_{shape}{extra}"

    def at_gpu_size(self) -> "WinCase":
        return replace(self, B=self.gpu[0], T=self.gpu[1]) if self.gpu else self

    @property
    def reward_rule(self) -> bool:
        return "mstdp" in self.rule

    def paths(self) -> dict:
        if self.kind == "dense":
            return dict(dense_staged=dense_mstdp_staged(self.B, self.nt), several_tiles=self.ns > 32,
                        tile_tail=self.ns % 32 != 0)
        if self.kind == "conv" and self.rule == "mstdp":
            return conv_mstdp_paths(self.geo, self.B)
        return {}


def _dense(rule, B, ns, nt, T=4, **kw):
    return WinCase("dense", rule, B, T, ns=ns, nt=nt, **kw)


def _conv(rule, B, geo, T=3, **kw):
    return WinCase("conv", rule, B, T, geo=geo, **kw)


def _local(rule, B, geo, T=3, **kw):
    return WinCase("local", rule, B, T, geo=geo, **kw)


def _listed_boundary(margin: int) -> ConvGeo:
    """A 1-channel convolution whose decoded source list has ``slist_cap - ns == margin`` (0: fits exactly)."""
    for h in range(40, 80):
        for w in range(40, 100):
            for co in (1, 2, 3):
                for kh in (2, 3, 4, 5):
                    g = ConvGeo(1, h, w, co, (kh, 3))
                    if conv_mstdp_paths(g, 1)["slist_margin"] == margin:
                        return g
    raise AssertionError(margin)


C4 = ConvGeo(1, 32, 32, 16, (5, 5))   # BASELINE config 4's convolution


def _window_cases():
    D, C, Lc = _dense, _conv, _local
    S = ("dense_staged", True)
    U = ("dense_staged", False)
    cs = [
        # dense MSTDP: the staging of the rule state switches at 32 B + 5 B nt + 16 <= 32 KB and B <= 768
        D("mstdp", 128, 784, 44, claims=(S,)),
        D("mstdp", 128, 784, 45, claims=(U,)),
        D("mstdp", 768, 33, 2, red="mean", claims=(S,)),
        D("mstdp", 769, 33, 2, claims=(U,)),
        D("mstdp", 1, 31, 9, red="mean", decay=True, claims=(S,)),
        D("mstdp", 3, 33, 17, reward=-0.5, bounds="inf", claims=(S,)),
        D("mstdp", 33, 784, 31, decay=True, reward=0.0, claims=(S,)),
        D("mstdp", 33, 31, 45, reward=-1.25, red="mean", claims=(S,)),
        D("mstdp", 200, 33, 45, decay=True, claims=(U,)),
        # MSTDPET (B = 1): staged up to nt = 6544
        D("mstdpet", 1, 33, 6544, T=3, claims=(S,)),
        D("mstdpet", 1, 33, 6545, T=3, claims=(U,)),
        D("mstdpet", 1, 63, 40, decay=True, reward=-0.5, claims=(S,)),
        # the MulticompartmentConnection forms
        D("mcc_mstdp", 5, 33, 20, decay=True, claims=(S,)),
        D("mcc_mstdpet", 1, 47, 20, reward=-0.5, claims=(S,)),
        # conv MSTDP
        C("mstdp", 2, _listed_boundary(0), claims=(("listed", True),)),
        C("mstdp", 2, _listed_boundary(-1), claims=(("listed", False), ("staged", True))),
        C("mstdp", 1, ConvGeo(1, 256, 12, 2, (3, 3)), claims=(("listed", True),)),
        C("mstdp", 1, ConvGeo(1, 257, 12, 2, (3, 3)), claims=(("listed", False), ("staged", True))),
        C("mstdp", 1, ConvGeo(1, 12, 256, 2, (3, 3)), claims=(("listed", True),)),
        C("mstdp", 1, ConvGeo(1, 12, 257, 2, (3, 3)), claims=(("listed", False), ("staged", True))),
        C("mstdp", 1, ConvGeo(1, 300, 200, 2, (3, 3), (1, 1)), p_src=0.05, claims=(("staged", False),)),
        C("mstdp", 2, ConvGeo(1, 100, 100, 1, (5, 5)), claims=(("stage_pm", False),)),
        C("mstdp", 3, ConvGeo(3, 12, 12, 4, (7, 7)), claims=(("cpc", 1), ("multi_channel", True))),
        C("mstdp", 3, ConvGeo(2, 9, 9, 3, (3, 3), (2, 2), (1, 1)), claims=(("unit_stride", False), ("listed", True))),
        C("mstdp", 2, ConvGeo(2, 257, 9, 3, (3, 3), (2, 1), (1, 1)), claims=(("unit_stride", False), ("listed", False))),
        C("mstdp", 4, ConvGeo(3, 10, 11, 2, (3, 2), (1, 1), (1, 0)), claims=(("multi_channel", True), ("listed", True))),
        C("mstdp", 3, ConvGeo(3, 260, 5, 2, (3, 3), (1, 1), (1, 1)),
          claims=(("multi_channel", True), ("listed", False))),
        C("mstdp", 1, ConvGeo(1, 9, 9, 2, (3, 3)), decay=True),
        C("mstdp", 31, ConvGeo(1, 9, 9, 2, (3, 3)), reward=-0.5),
        C("mstdp", 32, ConvGeo(1, 9, 9, 2, (3, 3))),
        C("mstdp", 33, ConvGeo(1, 9, 9, 2, (3, 3)), claims=(("shuffle_tail", True),)),
        C("mstdp", 65, ConvGeo(2, 7, 8, 2, (3, 3), (1, 1), (1, 1)), red="mean", claims=(("shuffle_tail", True),)),
        C("mstdp", 2, ConvGeo(1, 9, 9, 3, (3, 3)), red="mean", bounds="inf", gain_first=True),
        C("mstdp", 3, C4, gpu=(33, 6), claims=(("listed", True), ("stage_pm", True))),
        # PostPre / WeightDependentPostPre / Hebbian on a convolution
        C("postpre", 3, ConvGeo(2, 9, 9, 3, (3, 3), (2, 2), (1, 1))),
        C("postpre", 2, ConvGeo(3, 7, 8, 2, (3, 2), (1, 2), (0, 1)), nu_off=0),
        C("postpre", 4, ConvGeo(1, 8, 8, 2, (3, 3)), red="mean", decay=True, gain_first=True),
        C("wdep", 3, ConvGeo(2, 9, 9, 3, (3, 3), (2, 2), (1, 1)), nu_off=1),
        C("wdep", 2, ConvGeo(1, 10, 7, 2, (4, 3), (1, 1), (2, 1)), red="mean"),
        C("hebbian", 3, ConvGeo(2, 8, 9, 2, (2, 3), (2, 1), (1, 1)), bounds="inf"),
        C("hebbian", 2, ConvGeo(3, 6, 6, 2, (3, 3), (1, 1), (1, 1)), red="mean", decay=True),
        # LocalConnection2D rules (geo.cout = n_filters; no padding)
        Lc("postpre", 3, ConvGeo(1, 9, 9, 2, (3, 3), (2, 2))),
        Lc("postpre", 2, ConvGeo(3, 8, 9, 2, (3, 2), (2, 3)), red="mean"),
        Lc("wdep", 3, ConvGeo(3, 7, 7, 2, (3, 3), (2, 2))),
        Lc("wdep", 2, ConvGeo(1, 8, 6, 3, (2, 2), (2, 2)), nu_off=0, decay=True),
        Lc("hebbian", 2, ConvGeo(3, 6, 8, 2, (2, 3), (2, 2)), red="mean"),
        Lc("hebbian", 3, ConvGeo(1, 9, 8, 2, (3, 2), (3, 2)), bounds="inf"),
    ]
    return cs


WINDOW_CASES = _window_cases()


def draw_window(c: WinCase) -> dict:
    g = torch.Generator().manual_seed(7907 + 131 * c.B + 17 * c.T + 3 * len(c.name) + c.seed + sum(map(ord, c.name)))
    T, B = c.T, c.B
    if c.kind == "dense":
        src_shape, tgt_shape = (c.ns,), (1, 1, c.nt)   # [1, 1, nt]: the gain is a 1x1 convolution, not an nt x nt eye
        wshape = (c.ns, c.nt)
    elif c.kind == "conv":
        gg = c.geo
        src_shape, tgt_shape = (gg.cin, gg.hin, gg.win), (gg.cout, gg.hout, gg.wout)
        wshape = (gg.cout, gg.cin, *gg.k)
    else:
        gg = c.geo
        ho, wo = (gg.hin - gg.k[0]) // gg.s[0] + 1, (gg.win - gg.k[1]) // gg.s[1] + 1
        src_shape, tgt_shape = (gg.cin, gg.hin, gg.win), (gg.cout, ho, wo)
        wshape = (gg.cin, gg.cout * ho * wo, gg.k[0] * gg.k[1])
    nt = int(np.prod(tgt_shape))
    x_in = (torch.rand(T, B, *src_shape, generator=g) < c.p_src).to(torch.uint8)
    p_z = torch.linspace(0.3, 0.05, B).view(1, B, *([1] * len(tgt_shape)))
    z_in = (torch.rand(T, B, *tgt_shape, generator=g) < p_z).to(torch.uint8)
    if c.bounds == "finite":
        wmin, wmax = (0.0, 1.0) if c.rule in ("postpre", "wdep") else (-1.0, 1.0)
        w = wmin + (wmax - wmin) * (0.25 + 0.5 * torch.rand(*wshape, generator=g))
    else:
        wmin, wmax = -np.inf, np.inf
        w = torch.rand(*wshape, generator=g) - 0.4
    # learning rates scaled with the number of terms an update sums, so that the window moves the weights by a few
    # percent of their range at any B and size
    if c.kind == "dense":
        terms = 1.0
    elif c.kind == "conv":
        terms = 1.0 + 0.3 * c.geo.L
    else:
        terms = 1.0
    per_b = 1.0 if c.red == "mean" and not (c.kind == "conv" and c.rule == "mstdp") else float(B)
    scale = 1.0 / (per_b * terms * T)
    if c.reward_rule:
        nu0 = f32(0.2 * scale)
        nu1 = nu0
    else:
        nu0, nu1 = f32(0.3 * scale), f32(0.5 * scale)
        if c.nu_off == 0:
            nu0 = 0.0
        if c.nu_off == 1:
            nu1 = 0.0
    return dict(x_in=x_in, z_in=z_in, w=w.contiguous(), nu0=nu0, nu1=nu1, wmin=wmin, wmax=wmax,
                wd=0.0625 if c.decay else 0.0, a_plus=1.0, a_minus=-0.75, tc_plus=15.0, tc_minus=25.0, tc_e=10.0,
                tgt_shape=tgt_shape, src_shape=src_shape)


def run_kwargs(c: WinCase, d: dict) -> dict:
    return dict(reward=c.reward, a_plus=d["a_plus"], a_minus=d["a_minus"]) if c.reward_rule else {}


def build_window(ns_, c: WinCase, d: dict):
    """The network of a window case.  Returns (net, inputs)."""
    N, T_, Lr = ns_.nodes, ns_.topology, ns_.learning
    net = ns_.Network(dt=1.0, batch_size=c.B, learning=True)
    X = N.Input(shape=list(d["src_shape"]), traces=True)
    Z = N.Input(shape=list(d["tgt_shape"]))
    Y = N.LIFNodes(shape=list(d["tgt_shape"]), traces=True, thresh=Y_THRESH, refrac=0)
    net.add_layer(X, "X"); net.add_layer(Z, "Z"); net.add_layer(Y, "Y")
    red = {"sum": torch.sum, "mean": torch.mean}[c.red]
    nt = int(np.prod(d["tgt_shape"]))
    common = dict(wmin=d["wmin"], wmax=d["wmax"])
    if c.kind == "dense" and c.rule.startswith("mcc"):
        from bindsnet_b200.learning import MCC_learning as ML
        from bindsnet_b200.network.topology_features import Weight

        rule = ML.MSTDPET if c.rule == "mcc_mstdpet" else ML.MSTDP
        feat = Weight("w", d["w"].clone(), range=[d["wmin"], d["wmax"]], learning_rule=rule, nu=(d["nu0"], d["nu1"]),
                      reduction=red, decay=d["wd"])
        learned = T_.MulticompartmentConnection(X, Y, device="cpu", pipeline=[feat], tc_plus=d["tc_plus"],
                                                tc_minus=d["tc_minus"], tc_e_trace=d["tc_e"])
    elif c.kind == "dense":
        rule = {"mstdp": Lr.MSTDP, "mstdpet": Lr.MSTDPET}[c.rule]
        learned = T_.Connection(X, Y, w=d["w"].clone(), update_rule=rule, nu=(d["nu0"], d["nu1"]), reduction=red,
                                weight_decay=d["wd"], tc_plus=d["tc_plus"], tc_minus=d["tc_minus"], tc_e_trace=d["tc_e"],
                                **common)
    else:
        rule = {"mstdp": Lr.MSTDP, "postpre": Lr.PostPre, "wdep": Lr.WeightDependentPostPre, "hebbian": Lr.Hebbian}[c.rule]
        g = c.geo
        kw = dict(update_rule=rule, nu=(d["nu0"], d["nu1"]), reduction=red, weight_decay=d["wd"], **common)
        if c.rule == "mstdp":
            kw.update(tc_plus=d["tc_plus"], tc_minus=d["tc_minus"])
        if c.kind == "conv":
            learned = T_.Conv2dConnection(X, Y, kernel_size=g.k, stride=g.s, padding=g.p, w=d["w"].clone(), **kw)
        else:
            learned = T_.LocalConnection2D(X, Y, kernel_size=g.k, stride=g.s, n_filters=g.cout, **kw)
            with torch.no_grad():
                learned.w.copy_(d["w"])
    co = d["tgt_shape"][0]
    gain = T_.Conv2dConnection(Z, Y, kernel_size=1, stride=1, w=Z_GAIN * torch.eye(co).view(co, co, 1, 1))
    if c.gain_first:
        net.add_connection(gain, "Z", "Y"); net.add_connection(learned, "X", "Y")
    else:
        net.add_connection(learned, "X", "Y"); net.add_connection(gain, "Z", "Y")
    from bindsnet_b200.network.monitors import Monitor

    net.add_monitor(Monitor(Y, ["s"], time=c.T), "Ys")
    return net, {"X": d["x_in"], "Z": d["z_in"]}


def learned_weights(conn) -> torch.Tensor:
    if hasattr(conn, "pipeline"):
        return [f for f in conn.pipeline if type(f).__name__ == "Weight"][0].value
    return conn.w


def learned_rule(conn):
    if hasattr(conn, "pipeline"):
        return [f for f in conn.pipeline if type(f).__name__ == "Weight"][0].learning_rule
    return conn.update_rule


def window_state(net) -> dict:
    """Weights, Y's raster and the rule state (p_plus, p_minus, eligibility, eligibility trace), on the CPU."""
    conn = net.connections[("X", "Y")]
    ys = net.monitors["Ys"].get("s")
    out = {"w": learned_weights(conn).detach().cpu().clone(), "Ys": ys.cpu().reshape(ys.shape[0], -1).bool()}
    r = learned_rule(conn)
    for k in ("p_plus", "p_minus", "eligibility", "eligibility_trace"):
        v = getattr(r, k, None) if type(r).__name__ in ("MSTDP", "MSTDPET") else None
        if isinstance(v, torch.Tensor):
            out[k] = v.detach().cpu().float().clone()
    return out


def run_window(ns_, c: WinCase, d: dict, device: str = "cpu", spans=None):
    """Run the case (in windows of ``spans`` steps); returns (state, net)."""
    net, inputs = build_window(ns_, c, d)
    net.force_tier = 1
    if device != "cpu":
        net.to(device)
        inputs = {k: v.to(device) for k, v in inputs.items()}
    t0 = 0
    for span in spans or [c.T]:
        net.run(inputs={k: v[t0:t0 + span] for k, v in inputs.items()}, time=span, **run_kwargs(c, d))
        t0 += span
    return window_state(net), net


# ---- float64 restatements ----------------------------------------------------------------------------------------------

def _decay32(tc: float) -> float:
    """exp(-dt / tc) as the reference computes it: fp32 tensor arithmetic (learning.py:1564-1567)."""
    return float(torch.exp(-1.0 / torch.tensor(tc)))


def _im2col(v: torch.Tensor, g: ConvGeo) -> torch.Tensor:
    """The reference's im2col_indices: [B, cin * kh * kw, L] over the zero-padded input, with stride and WITHOUT
    dilation (rows in (ci, ky, kx) order, columns in (oy, ox) order); the target shape follows the reference's formula."""
    out = F.unfold(v, g.k, padding=g.p, stride=g.s)
    assert out.shape[2] == g.L, (out.shape, g)
    return out


def _local_unfold(v: torch.Tensor, g: ConvGeo, P: int, rule_view: bool) -> torch.Tensor:
    """LocalConnection2D's unfolded source.  ``rule_view`` (learning.py:280-309): the unfold [B, cin, ho, wo, kh, kw]
    reshaped as it lies in memory to [B, P, cin * K] and repeated n_filters times along dim 1: element (n', m) reads flat
    position (n' % P) * cin * K + m of the unfold — for cin > 1 not the window of n' in channel m // K.  Otherwise
    (topology.py:1731-1736) [B, cin, n_filters * P, K] with target n' reading window n' % P of every channel."""
    B = v.shape[0]
    u = v.unfold(2, g.k[0], g.s[0]).unfold(3, g.k[1], g.s[1]).contiguous()   # [B, cin, ho, wo, kh, kw]
    K = g.k[0] * g.k[1]
    if rule_view:
        return u.reshape(B, P, g.cin * K).repeat(1, g.cout, 1)
    return u.reshape(B, g.cin, P, K).repeat(1, 1, g.cout, 1)


def _stdp_apply(rule, w, err, U, Uabs, V, Vabs, d, pre_on, post_on, gam):
    """PostPre (learning.py:457-497 conv, :258-320 local), WeightDependentPostPre (:920-975, :717-791), Hebbian
    (:1348-1380, :1186-1250) from the batch-reduced pre / post sums U, V, then decay and clamp (:87-104)."""
    nu0, nu1, wmin, wmax = d["nu0"], d["nu1"], d["wmin"], d["wmax"]
    terms = w.abs() + err
    w0 = w
    if rule == "postpre":
        if pre_on:
            w = w - nu0 * U
            terms = terms + abs(nu0) * Uabs
        if post_on:
            w = w + nu1 * V
            terms = terms + abs(nu1) * Vabs
    elif rule == "wdep":
        upd = torch.zeros_like(w)
        if pre_on:
            upd = upd - nu0 * U * (w0 - wmin)
            terms = terms + abs(nu0) * Uabs * ((w0 - wmin).abs() + err)
        if post_on:
            upd = upd + nu1 * V * (wmax - w0)
            terms = terms + abs(nu1) * Vabs * ((wmax - w0).abs() + err)
        w = w + upd
    else:
        w = w + nu0 * U
        w = w + nu1 * V
        terms = terms + abs(nu0) * Uabs + abs(nu1) * Vabs
    return _decay_clamp(w, d, True), err + gam * terms


def _decay_clamp(w, d, clamp_rule: bool):
    if d["wd"]:
        w = w * (1.0 - d["wd"])
    if clamp_rule and (d["wmin"] != -np.inf or d["wmax"] != np.inf):
        w = w.clamp(d["wmin"], d["wmax"])
    return w


def ref_window(c: WinCase, d: dict, x_decay: float, y_decay: float):
    """The window replayed in float64.  Y's raster is Z's one step later (network.py:211-250 feeds the previous step's
    spikes).  Returns (w, bound, raster [T, B, nt] bool, traces) where traces = (p_plus, p_minus) with their bounds for
    the reward-modulated rules, else None."""
    f = torch.float64
    T, B = c.T, c.B
    w = d["w"].to(f)
    err = torch.zeros_like(w)
    nt = int(np.prod(d["tgt_shape"]))
    sY = torch.zeros(B, *d["tgt_shape"], dtype=f)
    xX = torch.zeros(B, *d["src_shape"], dtype=f)
    xY = torch.zeros(B, *d["tgt_shape"], dtype=f)
    dp, dm = _decay32(d["tc_plus"]), _decay32(d["tc_minus"])
    r, ap, am = c.reward, d["a_plus"], d["a_minus"]
    nu0 = d["nu0"]
    mean = c.red == "mean"
    ys = []
    g = c.geo
    if c.kind == "dense":
        pp, pm = torch.zeros(B, c.ns, dtype=f), torch.zeros(B, c.nt, dtype=f)
        sS_prev, sT_prev = torch.zeros(B, c.ns, dtype=f), torch.zeros(B, c.nt, dtype=f)
        et = torch.zeros_like(w)
        etabs = torch.zeros_like(w)
        pp_prev, pm_prev = pp.clone(), pm.clone()
    elif c.kind == "conv" and c.rule == "mstdp":
        pp_col = torch.zeros(B, g.K, g.L, dtype=f)
        pm = torch.zeros(B, g.cout, g.L, dtype=f)
        elig = torch.zeros(B, g.cout, g.K, dtype=f)
        eabs = torch.zeros_like(elig)
    for t in range(T):
        sX = d["x_in"][t].to(f)
        sY = d["z_in"][t - 1].to(f) if t > 0 else torch.zeros(B, *d["tgt_shape"], dtype=f)
        ys.append(sY.reshape(B, nt).bool())
        xX = torch.where(sX.bool(), torch.ones((), dtype=f), xX * x_decay)   # nodes.py:96-103
        xY = torch.where(sY.bool(), torch.ones((), dtype=f), xY * y_decay)
        if c.kind == "dense" and c.rule in ("mstdp", "mcc_mstdp"):
            # learning.py:1557-1574 (MCC_learning.py:515-548): w += nu0 * reduce_b(reward * eligibility(t - 1)), then
            # the traces, the new eligibility, decay, clamp
            gam = gamma(2 * T + B + 8)
            e = pp_prev.unsqueeze(2) * sT_prev.unsqueeze(1) + sS_prev.unsqueeze(2) * pm_prev.unsqueeze(1)
            ea = pp_prev.abs().unsqueeze(2) * sT_prev.unsqueeze(1) + sS_prev.unsqueeze(2) * pm_prev.abs().unsqueeze(1)
            upd, upd_abs = (r * e).sum(0), (abs(r) * ea).sum(0)
            if mean:
                upd, upd_abs = upd / B, upd_abs / B
            terms = w.abs() + err + abs(nu0) * upd_abs
            w = _decay_clamp(w + nu0 * upd, d, True)
            err = err + gam * terms
            sS, sT = sX.reshape(B, -1), sY.reshape(B, -1)
            pp = pp * dp + ap * sS
            pm = pm * dm + am * sT
            pp_prev, pm_prev, sS_prev, sT_prev = pp, pm, sS, sT
        elif c.kind == "dense":
            # MSTDPET learning.py:2229-2249 (MCC_learning.py:688-733), B = 1
            gam = gamma(5 * T + 8)
            de = _decay32(d["tc_e"])
            e = torch.outer(pp_prev[0], sT_prev[0]) + torch.outer(sS_prev[0], pm_prev[0])
            ea = torch.outer(pp_prev[0].abs(), sT_prev[0]) + torch.outer(sS_prev[0], pm_prev[0].abs())
            et = et * de + e / d["tc_e"]
            etabs = etabs * de + ea / d["tc_e"]
            coef = nu0 * 1.0 * r
            terms = w.abs() + err + abs(coef) * etabs
            w = _decay_clamp(w + coef * et, d, True)
            err = err + gam * terms
            sS, sT = sX.reshape(B, -1), sY.reshape(B, -1)
            pp = pp * dp + ap * sS
            pm = pm * dm + am * sT
            pp_prev, pm_prev, sS_prev, sT_prev = pp, pm, sS, sT
        elif c.kind == "conv" and c.rule == "mstdp":
            # learning.py:1972-2015 with the per-sample eligibility: the batch SUM whatever `reduction` says; P+ in
            # im2col space (padded taps stay 0), P- per output channel
            gam = gamma(2 * T + g.L + B + 8)
            upd, upd_abs = (r * elig).sum(0), (abs(r) * eabs).sum(0)
            terms = w.abs() + err + abs(nu0) * upd_abs.view(w.shape)
            w = _decay_clamp(w + nu0 * upd.view(w.shape), d, True)
            err = err + gam * terms
            s_col = _im2col(sX, g)
            sT = sY.reshape(B, g.cout, g.L)
            pp_col = pp_col * dp + ap * s_col
            pm = pm * dm + am * sT
            elig = torch.bmm(sT, pp_col.transpose(1, 2)) + torch.bmm(pm, s_col.transpose(1, 2))
            eabs = torch.bmm(sT, pp_col.abs().transpose(1, 2)) + torch.bmm(pm.abs(), s_col.transpose(1, 2))
        elif c.kind == "conv":
            gam = gamma(T + g.L + B + 8)
            s_col, x_col = _im2col(sX, g), _im2col(xX, g)
            xT, sT = xY.reshape(B, g.cout, g.L), sY.reshape(B, g.cout, g.L)
            U = torch.bmm(xT, s_col.transpose(1, 2)).sum(0).view(w.shape)      # learning.py:483-488
            V = torch.bmm(sT, x_col.transpose(1, 2)).sum(0).view(w.shape)      # :491-495
            if mean:
                U, V = U / B, V / B
            w, err = _stdp_apply(c.rule, w, err, U, U.abs(), V, V.abs(), d, c.rule == "hebbian" or d["nu0"] != 0.0,
                                 c.rule == "hebbian" or d["nu1"] != 0.0, gam)
        else:
            gam = gamma(T + B + 8)
            P = d["tgt_shape"][1] * d["tgt_shape"][2]
            s_u, x_u = _local_unfold(sX, g, P, True), _local_unfold(xX, g, P, True)   # [B, N, cin * K]
            U = (xY.reshape(B, nt, 1) * s_u).sum(0).reshape(w.shape)              # learning.py:312-314
            V = (sY.reshape(B, nt, 1) * x_u).sum(0).reshape(w.shape)              # :316-318
            if mean:
                U, V = U / B, V / B
            w, err = _stdp_apply(c.rule, w, err, U, U.abs(), V, V.abs(), d, c.rule == "hebbian" or d["nu0"] != 0.0,
                                 c.rule == "hebbian" or d["nu1"] != 0.0, gam)
    traces = None
    if c.reward_rule:
        if c.kind == "dense":
            traces = (pp, pm)
        else:
            # P+ back from im2col space to the source image (every unpadded tap of a position holds the same value)
            traces = (pp_src_from_col(pp_col, g, B), pm)
    return w, err, torch.stack(ys), traces


def pp_src_from_col(pp_col, g: ConvGeo, B: int):
    ones = torch.ones(B, g.cin, g.hin, g.win, dtype=pp_col.dtype)
    cnt = F.fold(_im2col(ones, g), (g.hin, g.win), g.k, padding=g.p, stride=g.s)
    tot = F.fold(pp_col, (g.hin, g.win), g.k, padding=g.p, stride=g.s)
    return torch.where(cnt > 0, tot / cnt.clamp(min=1), torch.zeros((), dtype=pp_col.dtype))


def ratio(w, w64, bound) -> float:
    return ke.ratio(w, w64, bound)


def check_window_bites(c: WinCase, d: dict, st: dict, interior_min: float = 0.5):
    """What the case claims to exercise, it does: weights changed, at least half of the changed ones strictly inside
    (wmin, wmax), a nonzero reward where one is claimed, Y spiked, and the claimed side of every switch holds."""
    w0, w = d["w"], st["w"]
    changed = w.contiguous().view(torch.int32) != w0.contiguous().view(torch.int32)
    assert changed.any(), f"{c.name}: no weight changed"
    if c.bounds == "finite":
        v = w[changed]
        inside = ((v > d["wmin"]) & (v < d["wmax"])).float().mean().item()
        assert inside >= interior_min, f"{c.name}: only {inside:.2f} of the changed weights are inside (wmin, wmax)"
    if c.reward_rule and c.reward != 0.0:
        assert d["nu0"] != 0.0
    assert st["Ys"].any(), f"{c.name}: Y never spiked"
    paths = c.paths()
    for k, side in c.claims:
        assert paths[k] == side, f"{c.name}: claims {k} = {side}, the mirror says {paths[k]}"


# ---- phase-1 gathers -----------------------------------------------------------------------------------------------

@dataclass(frozen=True)
class GatherCase:
    kind: str                     # "conv" or "local"
    B: int
    T: int
    geos: tuple                   # one or two ConvGeo (local: cout = n_filters); all into the same target
    claims: tuple = ()
    p_src: float = 0.3
    gpu: tuple = ()

    @property
    def name(self) -> str:
        return f"{self.kind}_b{self.B}_t{self.T}_" + "+".join(g.tag for g in self.geos)

    def at_gpu_size(self) -> "GatherCase":
        return replace(self, B=self.gpu[0], T=self.gpu[1]) if self.gpu else self

    def paths(self) -> dict:
        out = gather_paths(self.geos[0], self.B, self.kind == "local")
        out["two_convs"] = len(self.geos) > 1
        return out


_G = ConvGeo
_TWO_A = (_G(1, 12, 40, 2, (3, 3), (1, 1), (1, 1)), _G(1, 12, 40, 2, (5, 1), (1, 1), (2, 0)))


def _gather_cases():
    C = GatherCase
    return [
        # filter taps staged while a tile's channels hold <= 4096 taps: L = 1, 32 channels per tile, K = 128 / 130
        C("conv", 2, 3, (_G(2, 8, 8, 64, (8, 8)),), claims=(("st_taps_all", True), ("st_bits", True))),
        C("conv", 2, 3, (_G(2, 5, 13, 64, (5, 13)),), claims=(("st_taps_some_off", True), ("st_bits", True))),
        # source bits not staged: more than 4096 words (131 072 neurons) per sample
        C("conv", 1, 2, (_G(1, 363, 363, 2, (3, 3), (8, 8)),), p_src=0.1, gpu=(3, 3),
          claims=(("st_bits", False), ("word_straddle", True))),
        C("conv", 1, 2, (_G(2, 260, 260, 1, (4, 5), (9, 7), (1, 2)),), p_src=0.1, claims=(("st_bits", False),)),
        # funnel window up to kw = 32; tap by tap for kw = 33 (and for a dilated filter)
        C("conv", 2, 3, (_G(1, 6, 40, 2, (2, 32)),), claims=(("funnel", True), ("word_straddle", True))),
        C("conv", 2, 3, (_G(1, 6, 40, 2, (2, 33)),), claims=(("funnel", False),)),
        C("conv", 2, 3, (_G(2, 7, 45, 2, (2, 32), (1, 1), (0, 3)),), claims=(("funnel", True), ("word_straddle", True))),
        C("conv", 2, 3, (_G(2, 10, 9, 3, (3, 2), (1, 2), (1, 1), (2, 3)),), claims=(("funnel", False),)),
        # tap by tap (kw = 33) with the taps of a tile not staged (32 channels x 132 taps) and cin > 1
        C("conv", 2, 3, (_G(2, 2, 33, 64, (2, 33)),), claims=(("funnel", False), ("st_taps_some_off", True))),
        # two convolutions into one target, in both orders: only the first is staged, the second takes conv_geo
        C("conv", 3, 3, _TWO_A, claims=(("two_convs", True),)),
        C("conv", 3, 3, _TWO_A[::-1], claims=(("two_convs", True),)),
        C("conv", 2, 3, (_G(2, 9, 9, 2, (3, 3), (2, 2), (1, 1)), _G(1, 5, 5, 2, (1, 1))), claims=(("two_convs", True),)),
        # LocalConnection2D: rows of the window cut 32 bits at a time
        C("local", 2, 3, (_G(2, 4, 80, 2, (2, 32), (2, 16)),), claims=(("kw_over_32", False),)),
        C("local", 2, 3, (_G(2, 4, 80, 2, (2, 33), (2, 15)),), claims=(("kw_over_32", True),)),
        C("local", 2, 3, (_G(1, 5, 90, 3, (3, 40), (2, 25)),), claims=(("kw_over_32", True), ("word_straddle", True))),
        C("local", 2, 3, (_G(3, 6, 7, 2, (3, 3), (1, 2)),), claims=(("kw_over_32", False),)),
    ]


GATHER_CASES = _gather_cases()


def _local_shape(g: ConvGeo):
    return (g.cout, (g.hin - g.k[0]) // g.s[0] + 1, (g.win - g.k[1]) // g.s[1] + 1)


def draw_gather(c: GatherCase) -> dict:
    gen = torch.Generator().manual_seed(1299709 + c.B + sum(map(ord, c.name)))
    srcs, ws, bs = [], [], []
    for g in c.geos:
        srcs.append((torch.rand(c.T, c.B, g.cin, g.hin, g.win, generator=gen) < c.p_src).to(torch.uint8))
        if c.kind == "conv":
            ws.append(torch.rand(g.cout, g.cin, *g.k, generator=gen) - 0.3)
            bs.append(torch.rand(g.cout, generator=gen) - 0.5)
        else:
            co, ho, wo = _local_shape(g)
            ws.append(torch.rand(g.cin, co * ho * wo, g.k[0] * g.k[1], generator=gen) - 0.3)
            bs.append(None)
    return dict(srcs=srcs, ws=ws, bs=bs)


def build_gather(ns_, c: GatherCase, d: dict):
    N, T_ = ns_.nodes, ns_.topology
    net = ns_.Network(dt=1.0, batch_size=c.B, learning=False)
    g0 = c.geos[0]
    tgt = (g0.cout, g0.hout, g0.wout) if c.kind == "conv" else _local_shape(g0)
    Y = N.McCullochPitts(shape=list(tgt), thresh=1e9)
    inputs = {}
    for i, g in enumerate(c.geos):
        X = N.Input(shape=[g.cin, g.hin, g.win])
        net.add_layer(X, f"X{i}")
        inputs[f"X{i}"] = d["srcs"][i]
    net.add_layer(Y, "Y")
    for i, g in enumerate(c.geos):
        X = net.layers[f"X{i}"]
        if c.kind == "conv":
            conn = T_.Conv2dConnection(X, Y, kernel_size=g.k, stride=g.s, padding=g.p, dilation=g.d, w=d["ws"][i].clone(),
                                       b=d["bs"][i].clone())
        else:
            conn = T_.LocalConnection2D(X, Y, kernel_size=g.k, stride=g.s, n_filters=g.cout)
            with torch.no_grad():
                conn.w.copy_(d["ws"][i])
        net.add_connection(conn, f"X{i}", "Y")
    from bindsnet_b200.network.monitors import Monitor

    net.add_monitor(Monitor(Y, ["v"], time=c.T), "Yv")
    return net, inputs


def run_gather(ns_, c: GatherCase, d: dict, device: str = "cpu") -> torch.Tensor:
    """Y's voltages [T, B, n] (= its input every step)."""
    net, inputs = build_gather(ns_, c, d)
    net.force_tier = 1
    if device != "cpu":
        net.to(device)
        inputs = {k: v.to(device) for k, v in inputs.items()}
    net.run(inputs=inputs, time=c.T)
    v = net.monitors["Yv"].get("v")
    return v.detach().cpu().reshape(c.T, c.B, -1).clone()


def ref_local_compute(s: torch.Tensor, w: torch.Tensor, g: ConvGeo):
    """LocalConnection2D.compute (topology.py:1717-1740) in float64: per channel the window of target n' (window
    n' % P) times its own weights w[ci, n', :], summed over the window, then over the channels.  Bound:
    gamma_{cin (K + 1)} times the sum of the absolute terms."""
    sd, wd = s.to(torch.float64), w.to(torch.float64)
    co, ho, wo = _local_shape(g)
    u = _local_unfold(sd, g, ho * wo, False)          # [B, cin, N, K]
    out = (u * wd).sum(-1).sum(1)
    absum = (u * wd.abs()).sum(-1).sum(1)
    return out, gamma(g.cin * (g.k[0] * g.k[1] + 1)) * absum


def ref_gather(ns_, c: GatherCase, d: dict):
    """Every step's input of Y in float64: the sum of the connections' outputs for the PREVIOUS step's source spikes
    (step 0: silent sources).  Returns (v [T, B, n], bound)."""
    net, _ = build_gather(ns_, c, d)
    outs, bounds = [], []
    for t in range(c.T):
        tot, bnd = 0.0, 0.0
        for i, g in enumerate(c.geos):
            s = d["srcs"][i][t - 1] if t > 0 else torch.zeros_like(d["srcs"][i][0])
            conn = net.connections[(f"X{i}", "Y")]
            if c.kind == "conv":
                o, b = ke.ref_conv_compute(conn, s.bool(), d["ws"][i])
            else:
                o, b = ref_local_compute(s, d["ws"][i], g)
            o, b = o.reshape(c.B, -1), b.reshape(c.B, -1)
            tot, bnd = tot + o, bnd + b
        if len(c.geos) > 1:   # the one addition of the two connections' sums, on top of their own bounds
            bnd = bnd + gamma(2) * sum(
                (ke.ref_conv_compute(net.connections[(f"X{i}", "Y")], (d["srcs"][i][t - 1] if t > 0 else
                                     torch.zeros_like(d["srcs"][i][0])).bool(), d["ws"][i])[0].abs().reshape(c.B, -1)
                 for i in range(len(c.geos))))
        outs.append(tot)
        bounds.append(bnd)
    return torch.stack(outs), torch.stack(bounds)
