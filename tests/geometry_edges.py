"""Edge cases of the generic kernel's Conv1dConnection, Conv3dConnection and LocalConnection3D paths — phase 1's gathers
(``gather_conv1d``, ``gather_conv3d``, ``gather_local2d<.., true>``) and their staging, the learning phases
(``phase3_conv1d``, ``phase3_conv3d``, ``phase3_local3d``), the normalize phase (``normalize_conv_item``,
``normalize_local2d_item``) and their single-operator twins in csrc/snn_ops.cu — with plain float64 restatements of the
reference's formulas and Python mirrors of the conditions where the kernels change path (csrc/snn_phases.cuh).  Shared
by tests/test_geometry_edges.py (CPU: the oracle against float64, the emulated kernel against the oracle) and
tests/test_gpu_geometry_edges.py (the CUDA library).  No test functions here.

Window cases
------------
As in tests/learning_edges.py: the learned connection X -> Y is inserted first (``gain_first`` cases insert the gain
first, so the learned connection is not the input phase 1 stages).  Y (LIFNodes, ``thresh = 1e6``, ``refrac = 0``) is
driven only through a rule-less gain of 1e8 from an ``Input`` Z of Y's shape: a kernel-1 Conv1dConnection
(``1e8 * eye(cout)``) into a ``[cout, wout]`` target, a 1x1x1 Conv3dConnection into a Conv3dConnection's
``[F, d, h, w]`` target, and a kernel-1 LocalConnection3D with ``w[ci, f * P + p] = 1e8 [ci == f]`` into a
LocalConnection3D's target (the LocalConnection3D oracle holds no Conv3dConnection).  Y's raster is then Z's one step
later, whatever the learned weights round to.  The last sample of a batch never sees Z spike: its target traces stay
exactly zero and its targets silent (the warp-wide skips of ``phase3_local3d``).

A Conv3dConnection learns only learning.NoOp's decay and a zero-rate PostPre / WeightDependentPostPre (decay, then the
clamp): the reference's conv3d rules do not exist for non-zero rates.

Gather cases
------------
The connection feeds a ``McCullochPitts(thresh = 1e9)`` whose voltage is its input: a ``Monitor`` on ``v`` records every
step's gather, compared with a float64 convolution of the previous step's source spikes.

Single-operator cases
---------------------
``conn.compute(s)``, ``conn.update(learning=True)`` and ``conn.normalize()`` once each on layers whose ``s`` / ``x`` are
set by hand, as ``kernel_edges.run_update`` does: ``conv1d_compute_kernel``, ``conv3d_compute_kernel``,
``local3d_compute_kernel``, ``conv1d_update_kernel``, ``conv3d_update_kernel``, ``local3d_update_kernel``,
``conv_normalize_kernel`` and ``local3d_normalize_kernel``.  Before the normalize one filter (one row) is zeroed.

Error bound
-----------
With u = 2**-24 and gamma_k = k u / (1 - k u), a value computed from exact inputs by a sum of terms, each of which passes
through at most k roundings, differs from its exact value by at most gamma_k times the sum of the absolute values of its
terms (Higham, *Accuracy and Stability of Numerical Algorithms*, Lemma 3.1 and §3.1).  The rule constants (decay
factors, nu) are the fp32 values the kernels hold and are taken as exact inputs.

* A gather sums at most K taps (Conv1d: cin * kw, Conv3d: cin * kd * kh * kw) and the bias: gamma_{K+1} times the sum of
  the absolute terms.  A LocalConnection3D sums K = kd * kh * kw taps per channel, then the cin channel sums:
  gamma_{cin (K + 1)}.
* A trace after t steps carries t roundings (nodes.py:96-103).  One step of a Conv1d rule sums L = wout positions per
  sample and B samples (the mean adds a division), then ``nu * U`` (one), the pre and post updates (two), the decay
  (one), with spare roundings for WeightDependentPostPre's factors: T + L + B + 8 roundings per term.  A
  LocalConnection3D has one position per weight: T + B + 8.  NoOp's decay and the zero-rate Conv3d rules: one rounding.
* An error already in w is carried into the next step with a factor of magnitude <= 1 (see tests/learning_edges.py),
  so over a window the per-step bounds add up.
* A normalize sums a filter (a row) of K entries and scales by ``norm / sum``: K + 2 roundings relative to |w| times
  ``sum |w| / |sum w|``.  After a window, the error E carried in by the weights propagates as
  ``norm / |S| * (E_i + |w_i| sum E / (|S| - sum E))``; both add.
* A filter or row that sums to zero turns into inf / NaN in the reference (``norm / 0``): such entries must be
  non-finite exactly where float64 is, and of the same class (inf or NaN); they are compared by class, not by value.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, replace

import numpy as np
import torch
import torch.nn.functional as F

from kernel_edges import Y_THRESH, Z_GAIN, f32, gamma, ratio
from learning_edges import _decay_clamp, _stdp_apply

# csrc/snn_phases.cuh / snn_common.cuh
CONV_STAGE_WORDS = 4096     # SNN_CONV_STAGE_WORDS
CONV_STAGE_TAPS = 4096      # SNN_CONV_STAGE_TAPS
GEN_THREADS, TILE = 256, 32
LOCAL3D_EPL = 4             # SNN_LOCAL3D_EPL: a phase3_local3d unit covers 32 * 4 = 128 weights of a row

KINDS = ("conv1d", "conv3d", "local3d")


def nw(n: int) -> int:
    return (n + 31) // 32


@dataclass(frozen=True)
class Geo:
    """A Conv1dConnection ([cin, win] -> [cout, wout]), Conv3dConnection ([cin, d, h, w] -> [cout, d', h', w']) or
    LocalConnection3D ([cin, d, h, w] -> [cout = n_filters, d', h', w'], no padding).  ``src``, ``k``, ``s``, ``p``
    are per spatial axis (one for conv1d, three otherwise)."""
    kind: str
    cin: int
    src: tuple
    cout: int
    k: tuple
    s: tuple
    p: tuple = None

    @property
    def pad(self) -> tuple:
        return self.p if self.p is not None else (0,) * len(self.src)

    @property
    def out(self) -> tuple:
        return tuple((n - k + 2 * p) // s + 1 for n, k, s, p in zip(self.src, self.k, self.s, self.pad))

    @property
    def L(self) -> int:
        return int(np.prod(self.out))

    @property
    def K(self) -> int:
        """Taps of one (out, in) filter (conv) or of one row of a channel (local)."""
        return int(np.prod(self.k))

    @property
    def ns(self) -> int:
        return self.cin * int(np.prod(self.src))

    @property
    def nt(self) -> int:
        return self.cout * self.L

    @property
    def src_shape(self) -> tuple:
        return (self.cin, *self.src)

    @property
    def tgt_shape(self) -> tuple:
        return (self.cout, *self.out)

    @property
    def wshape(self) -> tuple:
        if self.kind == "local3d":
            return (self.cin, self.nt, self.K)
        return (self.cout, self.cin, *self.k)

    @property
    def tag(self) -> str:
        j = lambda t: "x".join(map(str, t))   # noqa: E731
        return (f"c{self.cin}x{j(self.src)}_o{self.cout}_k{j(self.k)}_s{j(self.s)}" +
                (f"_p{j(self.pad)}" if any(self.pad) else ""))


# ---- path mirrors: the C conditions, restated ------------------------------------------------------------------------

def _runs(g: Geo):
    """The tap runs the gathers cut out of the bit rows (gather_conv1d / gather_conv3d / gather_local2d<.., true>): for
    every output position, channel and kernel row the valid taps [kx_lo, kx_hi) in pieces of up to 32.  Yields
    (bit0 & 31, cnt, first) per piece; ``first``: the piece starts the row."""
    if g.kind == "conv1d":
        (win,), (kw,), (sw,), (pw,) = g.src, g.k, g.s, g.pad
        for ox in range(g.out[0]):
            ix0 = ox * sw - pw
            lo, hi = max(0, -ix0), min(kw, win - ix0)
            for ci in range(g.cin):
                for kx in range(lo, hi, 32):
                    yield (ci * win + ix0 + kx) & 31, min(32, hi - kx), kx == lo
        return
    (din, hin, win), (kd, kh, kw), (sd, sh, sw), (pd, ph, pw) = g.src, g.k, g.s, g.pad
    dout, hout, wout = g.out
    for oz in range(dout):
        for oy in range(hout):
            for ox in range(wout):
                iz0, iy0, ix0 = oz * sd - pd, oy * sh - ph, ox * sw - pw
                zs = range(max(0, -iz0), min(kd, din - iz0))
                ys = range(max(0, -iy0), min(kh, hin - iy0))
                lo, hi = max(0, -ix0), min(kw, win - ix0)
                for ci in range(g.cin):
                    for kz in zs:
                        for ky in ys:
                            row = ((ci * din + iz0 + kz) * hin + iy0 + ky) * win + ix0
                            for kx in range(lo, hi, 32):
                                yield (row + kx) & 31, min(32, hi - kx), kx == lo


def gather_paths(g: Geo, B: int) -> dict:
    """Phase 1's staging of the connection when it is the first conv-like input of its target, and the shapes of its
    tap runs.  ``st_bits``: True when the source bit rows are staged for every sample chunk (B * nw(ns) <= 4096), False
    when for none (nw(ns) > 4096 or, at B <= 32 where plan_units makes one chunk of B samples, B * nw(ns) > 4096), None
    when it depends on the grid.  ``st_taps_all`` / ``st_taps_some_off``: every 32-neuron tile stages the taps of its
    output channels ((co_hi - co_base + 1) * K <= 4096) / some tile does not (conv kinds only; a LocalConnection3D's
    weights are per target and never staged).  ``cross_word``: some run of taps crosses a 32-bit word (two words and a
    funnel shift); ``off0`` / ``off31``: some row starts at bit 0 / bit 31 of a word."""
    Snw = nw(g.ns)
    words = B * Snw
    st_bits = True if words <= CONV_STAGE_WORDS else (False if (B <= 32 or Snw > CONV_STAGE_WORDS) else None)
    out = dict(st_bits=st_bits, kw=g.k[-1], kw_over_32=g.k[-1] > 32)
    if g.kind != "local3d":
        K = g.cin * g.K
        taps = []
        for tile in range(nw(g.nt)):
            co_base = (tile * TILE) // g.L
            co_hi = min(g.nt - 1, tile * TILE + TILE - 1) // g.L
            taps.append((co_hi - co_base + 1) * K <= CONV_STAGE_TAPS)
        out.update(st_taps_all=all(taps), st_taps_some_off=not all(taps), st_taps_some_on=any(taps))
    cross, offs = False, set()
    for sft, cnt, first in _runs(g):
        cross |= sft + cnt > 32
        if first:
            offs.add(sft)
    out.update(cross_word=cross, off0=0 in offs, off31=31 in offs)
    # the padding cut of each axis (kx_lo / kx_hi, ky_*, kz_*): some window starts before or ends past the source
    names = ("x",) if g.kind == "conv1d" else ("z", "y", "x")
    for a, (n, k, s, p, o) in zip(names, zip(g.src, g.k, g.s, g.pad, g.out)):
        out[f"cut_{a}"] = p > 0 and (any(i * s - p < 0 for i in range(o)) or any(i * s - p + k > n for i in range(o)))
        out[f"s_gt_k_{a}"] = s > k
    out["pad"] = g.pad
    return out


def rule_paths(g: Geo, B: int) -> dict:
    """The switches of the learning phase.  phase3_conv1d: lanes per element ``grp`` = min(32, the power of two >= B),
    a short last group of samples (``group_tail``), the target row walked over more than one 32-bit word (``lq_loop``),
    a target row not word-aligned (``unaligned``), and the channel wrap of the reshape pairing (``wrap``: cin = 1,
    cin < L, cin = L, cin > L, where the while loop runs more than once).  phase3_local3d: the row of Mw = cin * K
    weights in segments of 128 (``segs``, ``seg_tail``) and the samples in groups of 32 (``b_groups``, ``b_tail``)."""
    if g.kind == "conv1d":
        grp = 1
        while grp < B and grp < 32:
            grp <<= 1
        L = g.L
        wrap = "cin=1" if g.cin == 1 else ("cin<L" if g.cin < L else ("cin=L" if g.cin == L else "cin>L"))
        return dict(grp=grp, group_tail=B % grp != 0, lq_loop=L > 32, unaligned=L % 32 != 0 and g.cout > 1, wrap=wrap,
                    L=L)
    if g.kind == "local3d":
        Mw = g.cin * g.K
        return dict(Mw=Mw, segs=-(-Mw // (32 * LOCAL3D_EPL)), seg_tail=Mw % (32 * LOCAL3D_EPL) != 0,
                    b_groups=-(-B // 32), b_tail=B % 32 != 0)
    return {}


def normalize_paths(g: Geo) -> dict:
    """The window's normalize phase runs nw(n_target) tiles of 256 threads over the filters (cout * cin) or rows
    (cin * n): ``multi_pass`` when a thread takes more than one."""
    items = g.cout * g.cin if g.kind != "local3d" else g.cin * g.nt
    return dict(multi_pass=items > nw(g.nt) * GEN_THREADS)


# ---- window cases ------------------------------------------------------------------------------------------------------

@dataclass(frozen=True)
class WinCase:
    rule: str                 # "postpre", "wdep", "hebbian", "noop" (conv3d: "noop", "postpre0", "wdep0" -- zero rate)
    B: int
    T: int
    geo: Geo
    red: str = "sum"
    nu_off: int = -1          # 0: nu0 = 0, 1: nu1 = 0
    norm: bool = False        # the connection has a norm: the window ends with the normalize phase
    zero_filter: bool = False # one filter (row) of w is zero: the normalize turns it into NaN
    gain_first: bool = False  # the gain is inserted before the learned connection (phase 1 stages the gain)
    p_src: float = 0.15
    gpu: tuple = ()           # (B, T) on the GPU where the CPU tier runs a smaller size
    claims: tuple = ()        # (switch, side) pairs of the path mirrors this case is there to reach

    @property
    def kind(self) -> str:
        return self.geo.kind

    @property
    def name(self) -> str:
        extra = "".join([f"_nu{self.nu_off}off" if self.nu_off >= 0 else "", "_norm" if self.norm else "",
                         "_zf" if self.zero_filter else "", "_gainfirst" if self.gain_first else ""])
        return f"{self.kind}_{self.rule}_b{self.B}_t{self.T}_{self.red}_{self.geo.tag}{extra}"

    def at_gpu_size(self) -> "WinCase":
        """The GPU runs every window at least 5 steps long."""
        return replace(self, B=self.gpu[0], T=self.gpu[1]) if self.gpu else replace(self, T=max(self.T, 5))

    @property
    def stdp(self) -> bool:
        return self.rule in ("postpre", "wdep", "hebbian")

    @property
    def pre_on(self) -> bool:
        return self.stdp and (self.rule == "hebbian" or self.nu_off != 0)

    @property
    def post_on(self) -> bool:
        return self.stdp and (self.rule == "hebbian" or self.nu_off != 1)

    def paths(self) -> dict:
        out = dict(gather_paths(self.geo, self.B), **rule_paths(self.geo, self.B))
        out["learned_first"] = not self.gain_first
        if self.norm:
            out.update(normalize_paths(self.geo))
        return out


def _c1(cin, win, cout, k, s=1, p=0):
    return Geo("conv1d", cin, (win,), cout, (k,), (s,), (p,))


def _c3(cin, src, cout, k, s=(1, 1, 1), p=(0, 0, 0)):
    return Geo("conv3d", cin, tuple(src), cout, tuple(k), tuple(s), tuple(p))


def _l3(cin, src, f, k, s=(1, 1, 1)):
    return Geo("local3d", cin, tuple(src), f, tuple(k), tuple(s))


# Conv3d: K = 16^3 = 4096 taps per (out, in) filter, L = 41 positions: tile 0 lies in channel 0 and stages its taps,
# tile 1 spans channels 0 and 1 (8192 taps) and does not, tile 2 lies in channel 1 and does
K4096 = _c3(1, (16, 16, 56), 2, (16, 16, 16))


def _window_cases():
    W = WinCase
    Bt, Bf = ("st_bits", True), ("st_bits", False)
    return [
        # ---- Conv1dConnection: batch groups, row lengths, the channel wrap, pre / post off, sum / mean
        W("postpre", 1, 4, _c1(1, 40, 2, 5, 1, 2), gpu=(1, 5), claims=(Bt, ("wrap", "cin=1"), ("lq_loop", True))),
        W("postpre", 2, 3, _c1(3, 20, 2, 3, 2, 1), nu_off=0, claims=(Bt, ("wrap", "cin<L"))),
        W("wdep", 3, 3, _c1(5, 9, 3, 4, 2, 1), red="mean", claims=(("wrap", "cin>L"), ("group_tail", True))),
        W("hebbian", 5, 3, _c1(7, 12, 2, 2, 5, 1), claims=(("wrap", "cin>L"), ("s_gt_k_x", True), ("cut_x", True))),
        W("postpre", 16, 3, _c1(2, 32, 2, 1), red="mean", claims=(("L", 32), ("group_tail", False))),
        W("wdep", 17, 3, _c1(2, 33, 2, 1), nu_off=1, claims=(("L", 33), ("group_tail", True), ("lq_loop", True))),
        W("hebbian", 31, 3, _c1(1, 70, 2, 31, 1, 15), red="mean", claims=(("L", 70), ("kw", 31), ("cross_word", True))),
        W("postpre", 32, 3, _c1(2, 40, 2, 32, 1, 16), norm=True, gpu=(32, 5), claims=(("kw", 32), ("group_tail", False))),
        W("wdep", 33, 3, _c1(1, 50, 2, 33, 2, 1), red="mean", claims=(("kw", 33), ("group_tail", True))),
        W("hebbian", 65, 3, _c1(2, 60, 2, 40, 5, 2), nu_off=0, claims=(("kw", 40), ("group_tail", True))),
        W("postpre", 3, 3, _c1(2, 100, 2, 65, 1, 3), red="mean", nu_off=1, norm=True, claims=(("kw", 65), ("L", 42))),
        W("wdep", 2, 4, _c1(2, 7, 1, 1), nu_off=0, claims=(("L", 7), ("wrap", "cin<L"))),
        W("hebbian", 2, 3, _c1(3, 9, 2, 3, 3), nu_off=1, red="mean", claims=(("wrap", "cin=L"),)),
        W("noop", 2, 3, _c1(2, 20, 3, 4, 2, 1), norm=True),
        W("postpre", 4, 3, _c1(2, 20, 2, 3, 1, 1), gain_first=True, claims=(("learned_first", False),)),
        # the staging of the bit rows and of the taps
        W("postpre", 32, 3, _c1(3, 1400, 2, 5, 50, 2), p_src=0.05, claims=(Bf,)),
        W("hebbian", 2, 3, _c1(2, 64, 64, 64), norm=True, claims=(("st_taps_all", True), ("kw", 64))),
        W("postpre", 2, 3, _c1(2, 65, 64, 65), claims=(("st_taps_some_off", True), ("kw", 65))),
        # more filters than one pass of the normalize phase: 32 x 9 > 1 tile x 256 threads
        W("postpre", 3, 3, _c1(9, 8, 32, 8), norm=True, claims=(("multi_pass", True), ("wrap", "cin>L"))),
        # ---- Conv3dConnection: NoOp decay and the zero-rate rules' decay + clamp; staging, padding cut per axis
        W("noop", 2, 3, K4096, norm=True, claims=(Bt, ("st_taps_some_off", True), ("st_taps_some_on", True))),
        W("postpre0", 10, 3, K4096, claims=(Bf, ("st_taps_some_off", True), ("st_taps_some_on", True))),
        W("wdep0", 3, 3, _c3(2, (5, 4, 6), 2, (3, 2, 3), (1, 1, 1), (1, 0, 0)), norm=True,
          claims=(Bt, ("cut_z", True), ("cut_y", False), ("cut_x", False), ("st_taps_all", True))),
        W("postpre0", 2, 3, _c3(2, (4, 6, 5), 3, (2, 3, 2), (1, 1, 1), (0, 1, 0)),
          claims=(("cut_z", False), ("cut_y", True), ("cut_x", False))),
        W("noop", 3, 4, _c3(1, (3, 4, 40), 2, (2, 2, 33), (1, 1, 2), (0, 0, 2)), norm=True, zero_filter=True,
          claims=(("cut_z", False), ("cut_y", False), ("cut_x", True), ("kw", 33))),
        W("wdep0", 2, 3, _c3(1, (9, 8, 10), 2, (2, 2, 2), (4, 3, 5), (1, 1, 1)),
          claims=(("s_gt_k_z", True), ("s_gt_k_x", True), ("cut_z", True))),
        W("noop", 2, 3, _c3(1, (2, 3, 6), 2, (1, 1, 1)), gain_first=True, claims=(("learned_first", False),)),
        # ---- LocalConnection3D: row segments of 128, sample groups of 32, normalize passes
        W("postpre", 1, 4, _l3(1, (3, 3, 4), 2, (1, 1, 1)), gpu=(1, 5), claims=(("Mw", 1), ("b_groups", 1))),
        W("wdep", 31, 3, _l3(1, (2, 2, 130), 2, (1, 1, 127), (1, 1, 3)), claims=(("Mw", 127), ("b_tail", True))),
        W("hebbian", 32, 3, _l3(2, (2, 5, 9), 2, (2, 4, 8)), red="mean", claims=(("Mw", 128), ("b_tail", False))),
        W("postpre", 33, 3, _l3(3, (1, 2, 45), 2, (1, 1, 43), (1, 1, 2)), nu_off=1, claims=(("Mw", 129), ("b_groups", 2))),
        W("wdep", 65, 3, _l3(1, (1, 2, 260), 2, (1, 1, 257), (1, 1, 3)), nu_off=0, red="mean",
          claims=(("Mw", 257), ("b_groups", 3), ("kw", 257))),
        W("hebbian", 3, 3, _l3(2, (3, 4, 35), 2, (2, 2, 32), (1, 2, 3)), nu_off=0, claims=(("kw", 32),)),
        W("noop", 2, 3, _l3(2, (2, 4, 6), 3, (1, 2, 3), (1, 2, 3)), norm=True, zero_filter=True),
        W("postpre", 5, 3, _l3(9, (1, 5, 5), 2, (1, 2, 2)), norm=True, claims=(("multi_pass", True),)),
        W("wdep", 4, 3, _l3(2, (2, 4, 5), 2, (1, 2, 2), (1, 2, 3)), red="mean", gain_first=True,
          claims=(("learned_first", False),)),
        W("postpre", 32, 3, _l3(1, (4, 4, 300), 2, (1, 1, 2), (1, 3, 100)), p_src=0.05, claims=(Bf,)),
    ]


WINDOW_CASES = _window_cases()


def _wbounds(c: WinCase):
    if c.rule in ("postpre0", "wdep0"):
        return 0.2, 0.8
    if c.rule in ("hebbian", "noop"):
        return -1.0, 1.0
    return 0.0, 1.0


def draw_window(c: WinCase) -> dict:
    g = c.geo
    gen = torch.Generator().manual_seed(6151 + 131 * c.B + 17 * c.T + sum(map(ord, c.name)))
    T, B = c.T, c.B
    x_in = (torch.rand(T, B, *g.src_shape, generator=gen) < c.p_src).to(torch.uint8)
    p_z = torch.linspace(0.3, 0.05, B)
    if B > 1:
        p_z[-1] = 0.0   # a sample whose targets never spike: its target traces stay exactly zero
    z_in = (torch.rand(T, B, *g.tgt_shape, generator=gen) < p_z.view(1, B, *([1] * len(g.tgt_shape)))).to(torch.uint8)
    wmin, wmax = _wbounds(c)
    if c.rule in ("hebbian", "noop"):
        w = 0.05 + 0.9 * torch.rand(*g.wshape, generator=gen)       # positive: the filter sums of normalize do not cancel
        if c.rule == "hebbian":
            w = w - 0.1
    elif c.rule in ("postpre0", "wdep0"):
        w = wmin + (wmax - wmin) * (0.02 + 0.96 * torch.rand(*g.wshape, generator=gen))
    else:
        w = wmin + (wmax - wmin) * (0.25 + 0.5 * torch.rand(*g.wshape, generator=gen))
    if c.zero_filter:
        (w.view(-1, g.K) if g.kind == "local3d" else w.view(g.cout * g.cin, -1))[1] = 0.0
    terms = 1.0 + 0.3 * g.L if g.kind == "conv1d" else 1.0
    per_b = 1.0 if c.red == "mean" else float(B)
    scale = 1.0 / (per_b * terms * T)
    nu0, nu1 = f32(0.3 * scale), f32(0.5 * scale)
    if c.nu_off == 0 or not c.stdp:
        nu0 = 0.0
    if c.nu_off == 1 or not c.stdp:
        nu1 = 0.0
    wd = 0.0625 if c.rule in ("noop", "postpre0", "wdep0") else 0.0
    # the norm: a filter's (row's) current sum on average, so that the normalize moves the weights by a little
    norm = float(w.reshape(-1, g.K).sum(1).mean()) if c.norm else None
    return dict(x_in=x_in, z_in=z_in, w=w.contiguous(), nu0=nu0, nu1=nu1, wmin=wmin, wmax=wmax, wd=wd, norm=norm)


def _learned(ns_, c, X, Y, d, w):
    T_, Lr = ns_.topology, ns_.learning
    g = c.geo
    rule = {"postpre": Lr.PostPre, "wdep": Lr.WeightDependentPostPre, "hebbian": Lr.Hebbian, "noop": Lr.NoOp,
            "postpre0": Lr.PostPre, "wdep0": Lr.WeightDependentPostPre}[c.rule]
    red = {"sum": torch.sum, "mean": torch.mean}[c.red]
    kw = dict(update_rule=rule, nu=(d["nu0"], d["nu1"]), reduction=red, weight_decay=d["wd"], wmin=d["wmin"],
              wmax=d["wmax"])
    if d["norm"] is not None:
        kw["norm"] = d["norm"]
    if g.kind == "conv1d":
        return T_.Conv1dConnection(X, Y, kernel_size=g.k[0], stride=g.s[0], padding=g.pad[0], w=w.clone(), **kw)
    if g.kind == "conv3d":
        return T_.Conv3dConnection(X, Y, kernel_size=g.k, stride=g.s, padding=g.pad, w=w.clone(), **kw)
    conn = T_.LocalConnection3D(X, Y, kernel_size=g.k, stride=g.s, n_filters=g.cout, **kw)
    with torch.no_grad():
        conn.w.copy_(w)
    return conn


def _gain(ns_, g: Geo, Z, Y):
    T_ = ns_.topology
    co = g.cout
    if g.kind == "conv1d":
        return T_.Conv1dConnection(Z, Y, kernel_size=1, w=Z_GAIN * torch.eye(co).view(co, co, 1))
    if g.kind == "conv3d":
        return T_.Conv3dConnection(Z, Y, kernel_size=1, w=Z_GAIN * torch.eye(co).view(co, co, 1, 1, 1))
    conn = T_.LocalConnection3D(Z, Y, kernel_size=1, stride=1, n_filters=co)
    w = torch.zeros(co, co, g.L)
    w[torch.arange(co), torch.arange(co)] = Z_GAIN   # w[ci, f * P + p, 0] = 1e8 where ci == f
    with torch.no_grad():
        conn.w.copy_(w.view(co, co * g.L, 1))
    return conn


def build_window(ns_, c: WinCase, d: dict):
    """The network of a window case.  Returns (net, inputs)."""
    N = ns_.nodes
    g = c.geo
    net = ns_.Network(dt=1.0, batch_size=c.B, learning=True)
    X = N.Input(shape=list(g.src_shape), traces=True)
    Z = N.Input(shape=list(g.tgt_shape))
    Y = N.LIFNodes(shape=list(g.tgt_shape), traces=True, thresh=Y_THRESH, refrac=0)
    net.add_layer(X, "X"); net.add_layer(Z, "Z"); net.add_layer(Y, "Y")
    learned, gain = _learned(ns_, c, X, Y, d, d["w"]), _gain(ns_, g, Z, Y)
    if c.gain_first:
        net.add_connection(gain, "Z", "Y"); net.add_connection(learned, "X", "Y")
    else:
        net.add_connection(learned, "X", "Y"); net.add_connection(gain, "Z", "Y")
    net.add_monitor(ns_.monitors.Monitor(Y, ["s", "v"], time=c.T), "Ys")
    return net, {"X": d["x_in"], "Z": d["z_in"]}


def run_window(ns_, c: WinCase, d: dict, device: str = "cpu"):
    """Run the case; returns ({"w", "Ys", "Yv"} on the CPU, net).  Y's voltages hold every step's gather of the learned
    connection (on top of the gain's), so comparing them bit for bit checks the learned gather and its staging too."""
    net, inputs = build_window(ns_, c, d)
    net.force_tier = 1
    if device != "cpu":
        net.to(device)
        inputs = {k: v.to(device) for k, v in inputs.items()}
    net.run(inputs=inputs, time=c.T)
    ys = net.monitors["Ys"].get("s")
    yv = net.monitors["Ys"].get("v")
    return {"w": net.connections[("X", "Y")].w.detach().cpu().clone(),
            "Ys": ys.cpu().reshape(ys.shape[0], -1).bool(), "Yv": yv.cpu().reshape(yv.shape[0], -1).clone()}, net


# ---- float64 restatements ----------------------------------------------------------------------------------------------

def _unfold_conv1d(v: torch.Tensor, g: Geo) -> torch.Tensor:
    """The reference's Conv1d rule view (learning.py:422-455): pad, unfold, reshape [B, -1, cin * k] — so a row l of
    the result holds elements of the [cin, L, k] unfold in memory order, not the window of position l."""
    B, (k,), (s,), (p,) = v.shape[0], g.k, g.s, g.pad
    return F.pad(v, (p, p)).unfold(-1, k, s).reshape(B, -1, g.cin * k)


def _unfold_local3d(v: torch.Tensor, g: Geo, rule_view: bool) -> torch.Tensor:
    """LocalConnection3D's unfolded source: three unfolds of the last three axes.  ``rule_view`` (learning.py:322-388):
    reshaped to [B, P, cin * K] and repeated n_filters times along dim 1; otherwise (topology.py:1866-1896)
    [B, cin, P, K] repeated along dim 2."""
    B = v.shape[0]
    u = v.unfold(-3, g.k[0], g.s[0]).unfold(-3, g.k[1], g.s[1]).unfold(-3, g.k[2], g.s[2])
    if rule_view:
        return u.reshape(B, g.L, g.cin * g.K).repeat(1, g.cout, 1)
    return u.reshape(B, g.cin, g.L, g.K).repeat(1, 1, g.cout, 1)


def rule_terms(g: Geo, sX, xX, sY, xY, mean: bool):
    """The batch-reduced pre / post sums U, V of one step (in w's shape, float64; every term is >= 0)."""
    B = sX.shape[0]
    if g.kind == "conv1d":
        U = torch.bmm(xY.reshape(B, g.cout, -1), _unfold_conv1d(sX, g)).sum(0)
        V = torch.bmm(sY.reshape(B, g.cout, -1), _unfold_conv1d(xX, g)).sum(0)
    else:
        s_u, x_u = _unfold_local3d(sX, g, True), _unfold_local3d(xX, g, True)   # [B, n, cin * K]
        U = (xY.reshape(B, g.nt, 1) * s_u).sum(0)      # bmm with the diagonal of x_tgt, learning.py:341-346
        V = (sY.reshape(B, g.nt, 1) * x_u).sum(0)
    if mean:
        U, V = U / B, V / B
    shape = (g.cout, g.cin, g.k[0]) if g.kind == "conv1d" else g.wshape
    return U.reshape(shape), V.reshape(shape)


def rule_step(c, g: Geo, w, err, U, V, d, gam):
    """One application of the case's rule (or NoOp's decay, or a zero-rate Conv3d rule's decay and clamp)."""
    if c.rule == "noop":
        return _decay_clamp(w, d, False), err + gam * (w.abs() + err)
    if c.rule in ("postpre0", "wdep0"):
        return _decay_clamp(w, d, True), err + gam * (w.abs() + err)
    return _stdp_apply(c.rule, w, err, U, U.abs(), V, V.abs(), d, c.pre_on, c.post_on, gam)


def ref_normalize(g: Geo, w: torch.Tensor, norm: float, err=None):
    """Conv1dConnection / Conv3dConnection.normalize (topology.py:665-676, :1004-1018): every (out, in) filter times
    ``norm / its sum``; LocalConnection3D.normalize (:1898-1909): every row of w viewed as [cin * n, K] likewise.  A
    zero sum gives inf / NaN.  ``err``: the error bound w carries in.  Returns (w', bound)."""
    w = w.to(torch.float64)
    rows = w.reshape(-1, g.K)
    S = rows.sum(1, keepdim=True)
    out = rows * (norm / S)
    E = torch.zeros_like(rows) if err is None else err.reshape(-1, g.K)
    SE = E.sum(1, keepdim=True)
    room = S.abs() - SE
    fac = norm / S.abs()
    prop = torch.where(room > 0, fac * (E + rows.abs() * SE / room.clamp(min=1e-300)),
                       torch.full_like(rows, math.inf))
    cond = torch.where(room > 0, (rows.abs().sum(1, keepdim=True) + SE) / room.clamp(min=1e-300),
                       torch.full_like(S, math.inf))
    bound = prop + gamma(g.K + 2) * (out.abs() + prop) * cond
    return out.reshape(w.shape), bound.reshape(w.shape)


def ref_window(c: WinCase, d: dict, x_decay: float, y_decay: float):
    """The window replayed in float64: Y's raster is Z's one step later (network.py:211-250 feeds the previous step's
    spikes); the traces follow nodes.py:96-103; the rule (or decay) every step; the normalize at the end.  Returns
    (w, bound, raster [T, B, nt] bool, (U seen non-zero, V seen non-zero))."""
    f = torch.float64
    g = c.geo
    T, B = c.T, c.B
    w = d["w"].to(f)
    err = torch.zeros_like(w)
    xX = torch.zeros(B, *g.src_shape, dtype=f)
    xY = torch.zeros(B, *g.tgt_shape, dtype=f)
    if c.stdp:
        gam = gamma(T + g.L + B + 8) if g.kind == "conv1d" else gamma(T + B + 8)
    else:
        gam = gamma(1)
    ys, u_seen, v_seen = [], False, False
    for t in range(T):
        sX = d["x_in"][t].to(f)
        sY = d["z_in"][t - 1].to(f) if t > 0 else torch.zeros(B, *g.tgt_shape, dtype=f)
        ys.append(sY.reshape(B, -1).bool())
        xX = torch.where(sX.bool(), torch.ones((), dtype=f), xX * x_decay)
        xY = torch.where(sY.bool(), torch.ones((), dtype=f), xY * y_decay)
        U = V = None
        if c.stdp:
            U, V = rule_terms(g, sX, xX, sY, xY, c.red == "mean")
            u_seen |= bool((U != 0).any())
            v_seen |= bool((V != 0).any())
        w, err = rule_step(c, g, w, err, U, V, d, gam)
    if d["norm"] is not None:
        w, err = ref_normalize(g, w, d["norm"], err)
    return w, err, torch.stack(ys), (u_seen, v_seen)


def check_window_bites(c: WinCase, d: dict, st: dict, seen, interior_min: float = 0.5):
    """What the case claims to exercise, it does: weights changed, at least half of the changed ones strictly inside
    (wmin, wmax), U and V non-zero somewhere where pre and post are on, Y spiked, and the claimed side of every
    switch holds."""
    w0, w = d["w"], st["w"]
    changed = w.contiguous().view(torch.int32) != w0.contiguous().view(torch.int32)
    assert changed.any(), f"{c.name}: no weight changed"
    v = w[changed]
    v = v[torch.isfinite(v)]
    inside = ((v > d["wmin"]) & (v < d["wmax"])).float().mean().item()
    assert inside >= interior_min, f"{c.name}: only {inside:.2f} of the changed weights are inside (wmin, wmax)"
    if c.pre_on:
        assert seen[0], f"{c.name}: the pre-synaptic sum U is zero throughout"
    if c.post_on:
        assert seen[1], f"{c.name}: the post-synaptic sum V is zero throughout"
    assert st["Ys"].any(), f"{c.name}: Y never spiked"
    check_claims(c)


def check_claims(c):
    paths = c.paths()
    for k, side in c.claims:
        assert paths[k] == side, f"{c.name}: claims {k} = {side}, the mirror says {paths[k]}"


# ---- phase-1 gathers -----------------------------------------------------------------------------------------------

@dataclass(frozen=True)
class GatherCase:
    B: int
    T: int
    geo: Geo
    claims: tuple = ()
    p_src: float = 0.3
    gpu: tuple = ()

    @property
    def kind(self) -> str:
        return self.geo.kind

    @property
    def name(self) -> str:
        return f"{self.kind}_b{self.B}_t{self.T}_{self.geo.tag}"

    def at_gpu_size(self) -> "GatherCase":
        return replace(self, B=self.gpu[0], T=self.gpu[1]) if self.gpu else self

    def paths(self) -> dict:
        return gather_paths(self.geo, self.B)


def _gather_cases():
    G = GatherCase
    return [
        # tap runs of kw = 1, 31, 32, 33, 40, 65: one word, one word or two, always two, more than one piece
        G(2, 3, _c1(2, 63, 2, 1), claims=(("kw", 1), ("off31", True))),
        G(2, 3, _c1(2, 70, 2, 31, 1, 3), claims=(("kw", 31), ("cross_word", True), ("off0", True), ("off31", True))),
        G(2, 3, _c1(1, 64, 3, 32, 1, 0), claims=(("kw", 32), ("off0", True), ("cross_word", True))),
        G(2, 3, _c1(3, 41, 2, 33, 2, 4), claims=(("kw", 33), ("kw_over_32", True), ("cut_x", True))),
        G(2, 3, _c1(2, 90, 2, 40, 5, 2), claims=(("kw", 40), ("s_gt_k_x", False))),
        G(2, 3, _c1(2, 100, 2, 65, 1, 3), claims=(("kw", 65), ("kw_over_32", True), ("off31", True))),
        G(3, 3, _c1(2, 30, 2, 2, 5, 1), claims=(("s_gt_k_x", True), ("cut_x", True))),
        G(1, 2, _c1(2, 70000, 2, 5, 5000, 2), p_src=0.05, claims=(("st_bits", False),)),
        G(2, 3, _c3(2, (2, 3, 70), 2, (1, 2, 31), (1, 1, 1), (0, 0, 1)), claims=(("kw", 31), ("off31", True), ("cross_word", True))),
        G(2, 3, _c3(1, (2, 2, 64), 2, (1, 1, 32), (1, 1, 1)), claims=(("kw", 32), ("off0", True))),
        G(2, 3, _c3(1, (2, 2, 70), 2, (2, 1, 40), (1, 1, 3), (1, 0, 2)), claims=(("kw", 40), ("kw_over_32", True))),
        G(2, 3, _c3(1, (1, 2, 66), 2, (1, 1, 65), (1, 1, 1)), claims=(("kw", 65), ("kw_over_32", True))),
        G(2, 3, _c3(2, (4, 5, 31), 2, (2, 2, 1), (1, 1, 1), (1, 1, 0)), claims=(("kw", 1), ("cut_z", True), ("cut_y", True))),
        G(1, 2, _c3(1, (64, 64, 40), 2, (2, 2, 2), (30, 30, 20)), p_src=0.05, claims=(("st_bits", False),)),
        G(2, 3, _l3(2, (3, 2, 63), 2, (2, 1, 1), (1, 1, 1)), claims=(("kw", 1), ("off31", True))),
        G(2, 3, _l3(1, (3, 3, 64), 2, (2, 2, 31), (1, 1, 1)), claims=(("kw", 31), ("cross_word", True), ("off0", True), ("off31", True))),
        G(2, 3, _l3(2, (3, 2, 70), 2, (2, 1, 32), (1, 1, 2)), claims=(("kw", 32), ("cross_word", True))),
        G(2, 3, _l3(1, (5, 2, 75), 2, (2, 1, 33), (2, 1, 3)), claims=(("kw", 33), ("kw_over_32", True))),
        G(2, 3, _l3(2, (1, 3, 80), 2, (1, 2, 40), (1, 1, 5)), claims=(("kw", 40), ("kw_over_32", True))),
        G(2, 3, _l3(1, (1, 2, 100), 3, (1, 1, 65), (1, 1, 7)), claims=(("kw", 65), ("kw_over_32", True))),
        G(1, 2, _l3(1, (64, 64, 40), 2, (2, 2, 2), (30, 30, 20)), p_src=0.05, claims=(("st_bits", False),)),
    ]


GATHER_CASES = _gather_cases()


def draw_gather(c: GatherCase) -> dict:
    g = c.geo
    gen = torch.Generator().manual_seed(1299721 + c.B + sum(map(ord, c.name)))
    src = (torch.rand(c.T, c.B, *g.src_shape, generator=gen) < c.p_src).to(torch.uint8)
    w = torch.rand(*g.wshape, generator=gen) - 0.3
    b = torch.rand(g.cout, generator=gen) - 0.5 if g.kind != "local3d" else None
    return dict(src=src, w=w, b=b)


def build_gather(ns_, c: GatherCase, d: dict):
    N, T_ = ns_.nodes, ns_.topology
    g = c.geo
    net = ns_.Network(dt=1.0, batch_size=c.B, learning=False)
    X = N.Input(shape=list(g.src_shape))
    Y = N.McCullochPitts(shape=list(g.tgt_shape), thresh=1e9)
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    if g.kind == "conv1d":
        conn = T_.Conv1dConnection(X, Y, kernel_size=g.k[0], stride=g.s[0], padding=g.pad[0], w=d["w"].clone(), b=d["b"].clone())
    elif g.kind == "conv3d":
        conn = T_.Conv3dConnection(X, Y, kernel_size=g.k, stride=g.s, padding=g.pad, w=d["w"].clone(), b=d["b"].clone())
    else:
        conn = T_.LocalConnection3D(X, Y, kernel_size=g.k, stride=g.s, n_filters=g.cout)
        with torch.no_grad():
            conn.w.copy_(d["w"])
    net.add_connection(conn, "X", "Y")
    net.add_monitor(ns_.monitors.Monitor(Y, ["v"], time=c.T), "Yv")
    return net, {"X": d["src"]}


def run_gather(ns_, c: GatherCase, d: dict, device: str = "cpu") -> torch.Tensor:
    """Y's voltages [T, B, n] (= its input every step)."""
    net, inputs = build_gather(ns_, c, d)
    net.force_tier = 1
    if device != "cpu":
        net.to(device)
        inputs = {k: v.to(device) for k, v in inputs.items()}
    net.run(inputs=inputs, time=c.T)
    return net.monitors["Yv"].get("v").detach().cpu().reshape(c.T, c.B, -1).clone()


def ref_compute(g: Geo, s: torch.Tensor, w: torch.Tensor, b):
    """The connection's compute in float64: F.conv1d / F.conv3d plus the bias (topology.py:640-656, :979-995), or
    LocalConnection3D's unfold * w summed over the window, then over the channels (:1866-1896).  Returns
    (out [B, n], bound)."""
    f = torch.float64
    sd, wd = s.to(f), w.to(f)
    B = s.shape[0]
    if g.kind == "local3d":
        u = _unfold_local3d(sd, g, False)    # [B, cin, n, K]
        out = (u * wd).sum(-1).sum(1)
        absum = (u * wd.abs()).sum(-1).sum(1)
        return out.reshape(B, -1), gamma(g.cin * (g.K + 1)) * absum.reshape(B, -1)
    conv = F.conv1d if g.kind == "conv1d" else F.conv3d
    p = g.pad[0] if g.kind == "conv1d" else g.pad
    s_ = g.s[0] if g.kind == "conv1d" else g.s
    bd = b.to(f)
    out = conv(sd, wd, bd, stride=s_, padding=p)
    absum = conv(sd, wd.abs(), bd.abs(), stride=s_, padding=p)
    return out.reshape(B, -1), gamma(g.cin * g.K + 1) * absum.reshape(B, -1)


def ref_gather(c: GatherCase, d: dict):
    """Every step's input of Y in float64: the connection's output for the PREVIOUS step's source spikes (step 0:
    silent sources).  Returns (v [T, B, n], bound)."""
    outs, bounds = [], []
    for t in range(c.T):
        s = d["src"][t - 1] if t > 0 else torch.zeros_like(d["src"][0])
        o, b = ref_compute(c.geo, s, d["w"], d["b"])
        outs.append(o)
        bounds.append(b)
    return torch.stack(outs), torch.stack(bounds)


# ---- single operators ------------------------------------------------------------------------------------------------

@dataclass(frozen=True)
class OpCase:
    rule: str
    B: int
    geo: Geo
    red: str = "sum"
    nu_off: int = -1
    gpu: tuple = ()           # (B,) on the GPU

    @property
    def kind(self) -> str:
        return self.geo.kind

    @property
    def name(self) -> str:
        return (f"{self.kind}_{self.rule}_b{self.B}_{self.red}_{self.geo.tag}" +
                (f"_nu{self.nu_off}off" if self.nu_off >= 0 else ""))

    def at_gpu_size(self) -> "OpCase":
        return replace(self, B=self.gpu[0]) if self.gpu else self

    stdp = WinCase.stdp
    pre_on = WinCase.pre_on
    post_on = WinCase.post_on

    def paths(self) -> dict:
        return dict(rule_paths(self.geo, self.B))


def _op_cases():
    O = OpCase
    return [
        O("postpre", 1, _c1(1, 40, 2, 5, 1, 2)),
        O("wdep", 3, _c1(5, 9, 3, 4, 2, 1), red="mean"),
        O("hebbian", 17, _c1(2, 70, 2, 3, 1, 1), nu_off=1),
        O("postpre", 33, _c1(3, 41, 2, 33, 2, 4), nu_off=0),
        O("noop", 5, _c1(2, 20, 3, 4, 2, 1)),
        O("noop", 2, _c3(2, (5, 4, 6), 2, (3, 2, 3), (1, 1, 1), (1, 0, 0))),
        O("postpre0", 4, _c3(1, (4, 5, 40), 2, (2, 2, 5), (1, 1, 2), (0, 0, 2))),
        O("wdep0", 3, _c3(2, (4, 6, 5), 3, (2, 3, 2), (2, 1, 1), (1, 1, 0))),
        O("postpre", 1, _l3(3, (1, 2, 45), 2, (1, 1, 43), (1, 1, 2))),
        O("wdep", 33, _l3(2, (2, 5, 9), 2, (2, 4, 8)), red="mean"),
        O("hebbian", 5, _l3(1, (2, 2, 130), 2, (1, 1, 127), (1, 1, 3)), nu_off=0),
        O("noop", 2, _l3(2, (2, 4, 6), 3, (1, 2, 3), (1, 2, 3))),
    ]


OP_CASES = _op_cases()


def draw_op(c: OpCase) -> dict:
    g = c.geo
    gen = torch.Generator().manual_seed(15485863 + c.B + sum(map(ord, c.name)))
    B = c.B

    def traces(shape):
        x = torch.rand(B, *shape, generator=gen)
        return torch.where(torch.rand(B, *shape, generator=gen) < 0.2, torch.zeros(()), x)   # exact zeros among them

    s_in = torch.rand(B, *g.src_shape, generator=gen) < 0.3
    s_in[0] = True                                       # every tap enters some output
    d = dict(s_in=s_in, s_src=torch.rand(B, *g.src_shape, generator=gen) < 0.25, x_src=traces(g.src_shape),
             s_tgt=torch.rand(B, *g.tgt_shape, generator=gen) < 0.15, x_tgt=traces(g.tgt_shape))
    if B > 1:
        d["x_tgt"][-1] = 0.0
        d["s_tgt"][-1] = False
    wmin, wmax = _wbounds(c)
    if c.rule in ("postpre0", "wdep0"):
        w = wmin + (wmax - wmin) * (0.02 + 0.96 * torch.rand(*g.wshape, generator=gen))
    elif c.rule in ("hebbian", "noop"):
        w = 0.05 + 0.9 * torch.rand(*g.wshape, generator=gen)
    else:
        w = wmin + (wmax - wmin) * (0.25 + 0.5 * torch.rand(*g.wshape, generator=gen))
    terms = 1.0 + 0.3 * g.L if g.kind == "conv1d" else 1.0
    scale = 1.0 / ((1.0 if c.red == "mean" else float(B)) * terms)
    nu0, nu1 = f32(0.3 * scale), f32(0.5 * scale)
    if c.nu_off == 0 or not c.stdp:
        nu0 = 0.0
    if c.nu_off == 1 or not c.stdp:
        nu1 = 0.0
    d.update(w=w.contiguous(), b=torch.rand(g.cout, generator=gen) - 0.5, nu0=nu0, nu1=nu1, wmin=wmin, wmax=wmax,
             wd=0.0625 if c.rule in ("noop", "postpre0", "wdep0") else 0.0, norm=float(w.reshape(-1, g.K).sum(1).mean()))
    return d


def zero_filter(g: Geo, w: torch.Tensor) -> torch.Tensor:
    """w with its second filter (row) zeroed."""
    w = w.clone()
    w.view(-1, g.K)[1] = 0.0
    return w


def run_op(ns_, c: OpCase, d: dict, device: str = "cpu"):
    """compute(s_in), then the rule's update once on the layers' s / x, then normalize() once after one filter (row) is
    zeroed.  Returns {"out", "w_upd", "w_norm"} on the CPU and the normalize's input."""
    N = ns_.nodes
    g = c.geo
    X, Y = N.Input(shape=list(g.src_shape), traces=True), N.LIFNodes(shape=list(g.tgt_shape), traces=True)
    for layer in (X, Y):
        layer.compute_decays(1.0)
        layer.set_batch_size(c.B)
    conn = _learned(ns_, c, X, Y, d, d["w"])
    if g.kind != "local3d":
        with torch.no_grad():
            conn.b.copy_(d["b"])
    X.s, X.x, Y.s, Y.x = (d[k].clone() for k in ("s_src", "x_src", "s_tgt", "x_tgt"))
    s = d["s_in"]
    if device != "cpu":
        for m in (X, Y, conn):
            m.to(device)
        s = s.to(device)
    out = conn.compute(s).detach().cpu().reshape(c.B, -1).clone()
    conn.update(learning=True)
    w_upd = conn.w.detach().cpu().clone()
    w_in = zero_filter(g, w_upd)
    with torch.no_grad():
        conn.w.copy_(w_in.to(conn.w.device))
    conn.normalize()
    return dict(out=out, w_upd=w_upd, w_norm=conn.w.detach().cpu().clone()), w_in


def ref_op_update(c: OpCase, d: dict):
    """One update in float64 from the given spikes and traces (exact inputs): the rule, or the decay (and the clamp of
    a zero-rate Conv3d rule).  Returns (w, bound, (U non-zero somewhere, V non-zero somewhere))."""
    g = c.geo
    f = torch.float64
    w = d["w"].to(f)
    U = V = None
    seen = (False, False)
    if c.stdp:
        U, V = rule_terms(g, d["s_src"].to(f), d["x_src"].to(f), d["s_tgt"].to(f), d["x_tgt"].to(f), c.red == "mean")
        seen = (bool((U != 0).any()), bool((V != 0).any()))
        gam = gamma(g.L + c.B + 8) if g.kind == "conv1d" else gamma(c.B + 8)
    else:
        gam = gamma(1)
    w1, err = rule_step(c, g, w, torch.zeros_like(w), U, V, d, gam)
    return w1, err, seen


# ---- comparisons ---------------------------------------------------------------------------------------------------

def assert_same(a: torch.Tensor, b: torch.Tensor, what: str):
    """Bit for bit, every NaN matching a NaN (the GPU's and the CPU's canonical NaN differ in sign and payload)."""
    a, b = a.float().contiguous(), b.float().contiguous()
    assert a.shape == b.shape, (what, a.shape, b.shape)
    na, nb = a.isnan(), b.isnan()
    ok = torch.equal(na, nb) and torch.equal(a[~na].view(torch.int32), b[~nb].view(torch.int32))
    if not ok:
        diff = (a.double() - b.double()).abs().nan_to_num(np.inf)
        raise AssertionError(f"{what}: {int(((a.view(torch.int32) != b.view(torch.int32)) & ~(na & nb)).sum())} entries "
                             f"differ, max |d| {float(diff.max()):.3e}")


def assert_within_bound(w: torch.Tensor, w64: torch.Tensor, bound: torch.Tensor, what: str) -> float:
    """|w - w64| <= bound where float64 is finite; where it is not, w is non-finite of the same class (inf or NaN, and
    the inf's sign)."""
    w = w.reshape(w64.shape)
    fin = torch.isfinite(w64)
    bad = ~fin
    if bool(bad.any()):
        assert torch.equal(w64[bad].isnan(), w[bad].isnan()), f"{what}: NaN where float64 has inf, or the other way"
        infs = w64[bad].isinf()
        assert torch.equal(w64[bad][infs], w[bad][infs].double()), f"{what}: an inf of the other sign"
    assert bool(torch.isfinite(w[fin]).all()), f"{what}: non-finite where float64 is finite"
    r = ratio(w[fin], w64[fin], bound[fin])
    assert r <= 1.0, f"{what}: |w - w_f64| reaches {r:.3g} x the rounding-error bound"
    return r
