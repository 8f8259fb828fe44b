"""Edge cases of the generic kernel's per-synapse tensor instantiation (``SYN``: ``phase3<true>``,
``phase3_mstdp_dense<true>``, ``apply_rule_syn`` / ``syn_at`` in csrc/snn_common.cuh, the single operator
``conn_update_kernel<true>`` in csrc/snn_ops.cu) and of its per-neuron parameter instantiation (``PN``: ``neuron_par``,
the ``PN`` branches of ``phase1`` / ``phase2`` / ``finalize_neuron`` and the theta rebuild at the end of the window in
csrc/snn_generic.cu), with plain float64 restatements of the reference's formulas and Python mirrors of the kernels'
path conditions.  Shared by tests/test_param_edges.py (CPU: the oracle against float64, the emulated kernel against
the oracle) and tests/test_gpu_param_edges.py (the CUDA library).  No test functions here.

The restatements are written from the reference (learning.py, nodes.py); the oracle that runs the cases is
tests/neuron_param_oracle.c, which includes the synapse-tensor oracle.

Error bounds
------------
u = 2**-24 and gamma_k = k u / (1 - k u) as in tests/kernel_edges.py: a value computed from exact inputs through at most
k roundings differs from the exact one by at most gamma_k times the sum of the absolute values of the terms it adds
(Higham, Lemma 3.1 and §3.1).

Synapses.  Per synapse (i, j) and step, with every rate, bound and trace read at (i, j):

* PostPre (learning.py:390-420): the target traces are scaled by ``nu0[j]`` before the bmm, so the kernel sums
  ``fl(x_tgt[b, j] nu0[j])`` over b; the post term sums ``fl(x_src[b, i] fl(s nu1[j]))`` (the product with s in {0, 1}
  is exact).  One rounding per term, B additions, the mean's division, the two updates of w and the decay: B + 5.
* WeightDependentPostPre (:626-653): ``(nu0 U) (w - wmin)`` and ``(nu1 V) (wmax - w)`` per element: three roundings
  per factor chain on top of the B + 1 of the reduced sums, two to accumulate ``upd`` and add it, one for the decay:
  B + 7.
* Hebbian (:1110-1136): ``nu reduce(bmm)``, ungated: B + 5.
* MSTDP (:1504-1574): ``nu0 reduce_b(reward e_b)``, e_b = p_plus (x) s_tgt + s_src (x) p_minus of the previous step
  (one rounding for the sum of the two products with a 0 / 1 factor, one for the reward): B + 6.
* MSTDPET (:2187-2249, B = 1): ``((nu0 dt) reward) e_trace``: three roundings for the coefficient and the product, two
  to update w and decay it.

Every bound therefore uses gamma_{B+8} per step, plus what the traces carry: an STDP trace after T steps is a product
of up to T decay factors (each product one rounding; the factors are the fp32 values the layers hold, inputs of the
restatement), an MSTDP p is a sum of decayed increments (two roundings a step), an MSTDPET eligibility trace adds three
more a step (multiply, divide, add) on top of its p's.  So the per-step constant is gamma_{B+T+8} (STDP),
gamma_{B+2T+8} (MSTDP) and gamma_{5T+10} (MSTDPET), times the sum of the absolute values of every term of the step.
An error already in w is carried with a factor of magnitude <= 1 (PostPre, Hebbian, MSTDP; |1 - nu0 U - nu1 V| <= 1
for the weight-dependent form at these rates; the decay; ``torch.clamp`` with tensor bounds is 1-Lipschitz in w, also
where ``wmin > wmax`` and it returns ``wmax``), so the window's bound is the sum of the per-step bounds, each taken
with |w| widened by the bound so far.

Neurons.  The float64 step uses ``decay = exp(-dt / tc_decay)`` (and ``theta_decay``, ``trace_decay``) evaluated in
float64 from the fp32 time constant; the fp32 factor the layer holds is torch's float32 ``exp`` of the rounded
``-dt / tc``: within 1 ulp (2u relative) of the exact exponential of its argument, whose rounding moves the result
by at most u dt / tc <= u relative.  So |decay_32 - decay_64| <= 3u decay_64 (asserted on every case's layers).  One
LIF / AdaptiveLIF / DiehlAndCook step (nodes.py:500-529, 921-946, 1069-1110)

    v' = fl(fl(fl(decay fl(v - rest)) + rest) + gate x)

has four roundings, each at most u times the magnitude of its result, plus the decay's error 3u |decay (v - rest)|:

    e' = decay (1 + 3u) e + gamma_5 (|decay (v - rest)| + |rest| + |x| + |v'|) + 3u |decay (v - rest)|

where e is the bound v carries in and x (the input, a sum of weights that are multiples of 1/8 over at most a few
hundred spikes) is exact in fp32.  A reset sets e = 0 (``reset`` is exact), the lower bound is 1-Lipschitz.  The
threshold compare is exact for LIF (``v >= thresh``) and compares with fl(thresh + theta) for DC / AdaptiveLIF: the
margin required at every neuron-step is e + e_theta + u |thresh + theta|.  theta (shared by the batch) follows
``theta *= theta_decay; theta += theta_plus * count``: e_theta' = theta_decay (1 + 3u) e_theta + (3u + gamma_3)
(|theta theta_decay| + |theta_plus count| + |theta'|).  Traces: ``x *= trace_decay`` then ``x += fl(scale s)``
(additive) or ``x = scale`` on a spike: e_x' = trace_decay (1 + 3u) e_x + (3u + gamma_3) (|x trace_decay| + |scale| +
|x'|), 0 after a non-additive spike.  Refractory counts are small integers: exact.

The neuron dynamics are teacher-forced: the float64 voltages are stepped with the oracle's spikes (and, for
``one_spike``, its winners), every neuron-step's float64 voltage must lie farther than the margin from its threshold
(so the raster does not depend on rounding), and the float64 raster must equal the oracle's.
"""
from __future__ import annotations

from dataclasses import dataclass, replace

import numpy as np
import torch

from kernel_edges import EAGER_B, XT_STAGED_MAX_B, f32, gamma

U32 = 2.0 ** -24
P3_MAXEV = 16            # SNN_P3_MAXEV (snn_phases.cuh)
GEN_WARPS = 8            # SNN_GEN_THREADS / 32
EMU_CAP = 6              # co-resident CTAs of the emulated 3-SM device (2 per SM, tests/emu)
DECAY_REL = 3 * U32      # |decay_32 - decay_64| / decay_64, see the module docstring
MSTDP_SMEM = 4 * GEN_WARPS * 32 * 32   # bytes phase3_mstdp_dense may stage (its `staged` test, snn_phases.cuh)
Y_THRESH, Z_GAIN = 1.0e6, 1.0e8        # as in tests/kernel_edges.py: Y spikes exactly one step after Z
PN_ROWS = ("thresh", "rest", "decay", "theta_plus", "theta_decay", "trace_decay", "trace_scale")   # SNN_PN_* order


def _ceil(a, b):
    return (a + b - 1) // b


# ---- path mirrors -------------------------------------------------------------------------------------------------

def p3_row_chunks(ns: int, nt: int, cap: int) -> int:
    """plan_units (snn_generic.cu): row chunks per target tile of a dense STDP connection."""
    rc = min(_ceil(cap, _ceil(nt, 32)), _ceil(_ceil(ns, 32), GEN_WARPS))
    return max(rc, 1)


def sample_chunks(B: int, total_items: int, cap: int) -> int:
    """plan_units: the number of sample chunks (N.nch) of phases 1 / 2."""
    nch = _ceil(B, 4 * GEN_WARPS)
    while nch > 1 and total_items * nch > 16 * cap:
        nch -= 1
    cs = _ceil(B, nch)
    return _ceil(B, cs)


def mstdp_staged(B: int, nt: int) -> bool:
    """phase3_mstdp_dense's `staged` (snn_phases.cuh): the trace tile fits (B <= 768) and the whole rule state does."""
    return 32 * 4 * B <= 96 * 1024 and B * 32 + B * nt * 5 + 16 <= MSTDP_SMEM


def tile_events(s_tgt: torch.Tensor) -> int:
    """The largest number of samples with a post-synaptic event in one 32-column tile."""
    B, nt = s_tgt.shape
    pad = torch.zeros(B, _ceil(nt, 32) * 32, dtype=torch.bool)
    pad[:, :nt] = s_tgt
    return int(pad.view(B, -1, 32).any(2).sum(0).max())


# ---- synapse cases ------------------------------------------------------------------------------------------------

STDP = ("postpre", "wdep", "hebbian")
SYN_RULES = STDP + ("mstdp", "mstdpet")


@dataclass(frozen=True)
class SynCase:
    rule: str
    B: int
    ns: int
    nt: int
    T: int = 4
    red: str = "sum"
    lo: str = "full"          # wmin: full / tgt / src / tfull (a transposed view, copied by the host) / scalar
    hi: str = "tgt"           # wmax: likewise
    nu: str = "tgt"           # both rates: full / tgt / src / one / tfull / scalar
    decay: bool = False       # weight decay 0.0625 (factor 0.9375, exact)
    inf: bool = False         # infinite bound elements (not for the weight-dependent rule)
    nu_zero: int = -1         # 0 / 1: nu[k] is all zero (the rate gate is off)
    outside: bool = False     # user weights outside their bounds, an element with wmin > wmax and one with wmin == wmax
    events: str = "rand"      # "all": every sample's Y spikes in column 0 at every step (B events in tile 0)
    reward: float = 1.0
    pn: bool = False          # also a per-neuron population on X: the <SYN, PN> instantiation
    op: bool = False          # the single operator connection.update() (conn_update_kernel<true>) instead of a window
    seed: int = 0
    claims: tuple = ()
    gpu: tuple = ()           # (B, T, ns) on the GPU where the CPU file runs a smaller case

    @property
    def name(self) -> str:
        extra = "".join([f"_nu{self.nu_zero}zero" if self.nu_zero >= 0 else "", "_decay" if self.decay else "",
                         "_inf" if self.inf else "", "_out" if self.outside else "", "_allev" if self.events == "all" else "",
                         f"_r{self.reward:g}" if self.reward != 1.0 else "", "_pn" if self.pn else "",
                         f"_s{self.seed}" if self.seed else ""])
        head = "op" if self.op else f"T{self.T}"
        return f"{self.rule}_{head}_b{self.B}_{self.ns}x{self.nt}_{self.red}_lo{self.lo}_hi{self.hi}_nu{self.nu}{extra}"

    def at_gpu_size(self) -> "SynCase":
        if not self.gpu:
            return replace(self, T=max(self.T, 5)) if not self.op else self
        B, T, ns = self.gpu
        return replace(self, B=B, T=T, ns=ns)

    @property
    def stdp(self) -> bool:
        return self.rule in STDP


def _syn_cases():
    S = SynCase
    return [
        # phase3<true>: the 16 event slots of a tile, eager prefetch, staged / unstaged target traces, row chunks
        S("postpre", 1, 40, 33, T=6, lo="tgt", hi="src", nu="tgt", claims=(("slots_only", True), ("eager", False))),
        S("postpre", 16, 48, 33, events="all", lo="full", hi="tgt", nu="tgt", outside=True,
          claims=(("overflow", False), ("max_events", 16), ("full_clamp0", True))),
        S("postpre", 17, 48, 33, events="all", lo="src", hi="full", nu="tgt", claims=(("overflow", True), ("max_events", 17))),
        S("wdep", 17, 48, 95, events="all", lo="full", hi="full", nu="full", outside=True, claims=(("overflow", True),)),
        S("hebbian", 20, 40, 33, events="all", lo="full", hi="full", nu="src", inf=True, claims=(("overflow", True),)),
        S("postpre", 63, 300, 33, T=3, lo="full", hi="tgt", nu="tgt", gpu=(63, 5, 784),
          claims=(("eager", False), ("row_chunks", True))),
        S("postpre", 64, 300, 33, T=3, lo="tgt", hi="full", nu="one", gpu=(64, 5, 784), claims=(("eager", True), ("row_chunks", True))),
        S("wdep", 64, 48, 64, T=3, lo="src", hi="tgt", nu="src", red="mean", claims=(("eager", True), ("nt_tail", False))),
        S("hebbian", 65, 300, 95, T=3, lo="tfull", hi="src", nu="tfull", claims=(("row_chunks", True), ("copied", True))),
        S("postpre", 768, 48, 33, T=3, lo="full", hi="scalar", nu="tgt", claims=(("staged", True),)),
        S("postpre", 769, 48, 33, T=3, lo="full", hi="tgt", nu="tgt", outside=True, claims=(("staged", False),)),
        S("wdep", 769, 40, 95, T=3, lo="tgt", hi="full", nu="tgt", decay=True, claims=(("staged", False), ("full_decay", True))),
        S("hebbian", 768, 40, 33, T=3, lo="tgt", hi="tgt", nu="full", red="mean", claims=(("staged", True),)),
        # gates, forms, infinite elements, the step-0 clamp, decay
        S("postpre", 4, 40, 33, lo="full", hi="full", nu="tgt", inf=True, outside=True, claims=(("full_clamp0", True),)),
        S("postpre", 5, 48, 33, lo="tgt", hi="tgt", nu="tgt", nu_zero=0, claims=(("pre_on", False), ("post_on", True))),
        S("postpre", 5, 48, 33, lo="src", hi="src", nu="tgt", nu_zero=1, claims=(("pre_on", True), ("post_on", False))),
        S("wdep", 6, 48, 33, lo="full", hi="src", nu="full", nu_zero=0, outside=True, claims=(("pre_on", False),)),
        S("wdep", 6, 40, 33, lo="tgt", hi="full", nu="one", nu_zero=1, decay=True, claims=(("post_on", False), ("full_decay", True))),
        S("wdep", 3, 40, 33, lo="full", hi="full", nu="tgt", outside=True),
        S("hebbian", 4, 40, 95, lo="src", hi="tgt", nu="one", inf=True, decay=True),
        S("hebbian", 3, 48, 33, lo="full", hi="full", nu="tgt", nu_zero=0, outside=True),
        S("postpre", 3, 40, 33, lo="tfull", hi="tfull", nu="one", red="mean", outside=True, claims=(("copied", True),)),
        # ns = 1 and nt = 1: the host's stride test collapses a full tensor into a per-target / per-source one
        S("wdep", 4, 1, 40, lo="full", hi="full", nu="full", claims=(("collapsed", True),)),
        S("hebbian", 4, 40, 1, T=6, lo="full", hi="full", nu="full", claims=(("collapsed", True),)),
        S("postpre", 4, 1, 33, lo="full", hi="tgt", nu="tgt", claims=(("collapsed", True),)),
        # phase3_mstdp_dense<true>: staged vs unstaged through B * nt, sum and mean, negative reward, zero rates
        S("mstdp", 1, 40, 33, T=6, lo="full", hi="full", nu="full", claims=(("mstdp_staged", True),)),
        S("mstdp", 4, 40, 33, T=5, lo="src", hi="tgt", nu="src", red="mean", reward=-0.5, outside=True),
        S("mstdp", 64, 40, 95, T=3, lo="full", hi="src", nu="full", claims=(("mstdp_staged", True),)),
        S("mstdp", 65, 40, 95, T=3, lo="tgt", hi="full", nu="tgt", red="mean", claims=(("mstdp_staged", False),)),
        S("mstdp", 3, 40, 2200, T=3, lo="full", hi="full", nu="full", claims=(("mstdp_staged", False),)),
        S("mstdp", 2, 40, 33, T=4, lo="tgt", hi="tgt", nu="one", decay=True, inf=True),
        S("mstdpet", 1, 40, 33, T=10, lo="full", hi="full", nu="full", outside=True),
        S("mstdpet", 1, 48, 95, T=6, lo="src", hi="tgt", nu="src", reward=-0.75, decay=True),
        S("mstdpet", 1, 40, 33, T=5, lo="tgt", hi="full", nu="tgt", inf=True),
        # the <SYN, PN> instantiation
        S("postpre", 20, 48, 33, lo="full", hi="tgt", nu="tgt", events="all", pn=True, claims=(("overflow", True),)),
        S("mstdp", 3, 40, 33, T=4, lo="full", hi="full", nu="full", pn=True),
        # the single operator connection.update() (phase3<true> at t = 0: the clamp pass is full)
        S("postpre", 1, 40, 33, op=True, lo="full", hi="tgt", nu="tgt", outside=True),
        S("postpre", 17, 48, 95, op=True, events="all", lo="src", hi="full", nu="tgt", claims=(("overflow", True),)),
        S("postpre", 16, 48, 33, op=True, events="all", lo="tgt", hi="tgt", nu="one", claims=(("overflow", False), ("max_events", 16))),
        S("wdep", 63, 300, 33, op=True, lo="full", hi="full", nu="full", outside=True, claims=(("eager", False), ("warp_loops", True))),
        S("wdep", 64, 48, 64, op=True, lo="tfull", hi="src", nu="tgt", claims=(("eager", True), ("copied", True), ("nt_tail", False))),
        S("hebbian", 769, 48, 33, op=True, lo="full", hi="full", nu="src", inf=True, claims=(("staged", False),)),
        S("postpre", 768, 48, 33, op=True, lo="full", hi="tgt", nu="tgt", claims=(("staged", True),)),
        S("postpre", 769, 40, 33, op=True, lo="tgt", hi="full", nu="tgt", decay=True, nu_zero=0, claims=(("staged", False), ("pre_on", False))),
        S("hebbian", 5, 40, 33, op=True, lo="full", hi="full", nu="full", nu_zero=1, outside=True),
        S("wdep", 4, 1, 33, op=True, lo="full", hi="full", nu="full", nu_zero=1, claims=(("collapsed", True), ("post_on", False))),
        # one-element bound tensors: the host reads them into the scalar fields (a bound tensor is per-synapse only with
        # more than one element), beside tensors of the other forms
        S("wdep", 5, 40, 33, lo="one", hi="full", nu="tgt", outside=True),
        S("postpre", 4, 40, 33, op=True, lo="src", hi="one", nu="one", outside=True),
    ]


SYN_CASES = _syn_cases()


def _rates_scale(c: SynCase) -> tuple:
    base = {"postpre": (0.02, 0.03), "wdep": (0.05, 0.05), "hebbian": (0.004, 0.004), "mstdp": (0.05, 0.05), "mstdpet": (0.05, 0.05)}[c.rule]
    k = 1.0 if c.red == "mean" else 1.0 / c.B
    return base[0] * k, base[1] * k


def _tensor_of(form: str, full: torch.Tensor, g: torch.Generator, ns: int, nt: int):
    """A tensor of the given form whose broadcast to [ns, nt] is taken from ``full``'s row 0 / column 0 / element 0."""
    if form == "full":
        return full.clone()
    if form == "tfull":
        return full.t().contiguous().t()          # strides (1, ns): the host copies it to a contiguous [ns, nt]
    if form == "tgt":
        return full[0].clone()
    if form == "src":
        return full[:, :1].clone()
    if form == "one":
        return full.reshape(-1)[:1].clone()
    raise ValueError(form)


def bcast(t, ns, nt) -> torch.Tensor:
    """A bound or rate as float64 [ns, nt]."""
    if isinstance(t, torch.Tensor):
        return t.to(torch.float64).expand(ns, nt).clone()
    return torch.full((ns, nt), float(t), dtype=torch.float64)


def draw_syn(c: SynCase) -> dict:
    g = torch.Generator().manual_seed(2027 + 7919 * c.seed + 131 * c.B + 17 * c.ns + c.nt + SYN_RULES.index(c.rule))
    B, ns, nt, T = c.B, c.ns, c.nt, max(c.T, 1)
    x_in = (torch.rand(T, B, ns, generator=g) < 0.15).to(torch.uint8)
    z_in = (torch.rand(T, B, nt, generator=g) < torch.linspace(0.03, 0.2, B).view(1, B, 1)).to(torch.uint8)
    if c.events == "all":
        z_in[:, :, 0] = 1
    lo = -0.2 - 0.8 * torch.rand(ns, nt, generator=g)
    hi = 0.3 + 0.8 * torch.rand(ns, nt, generator=g)
    if c.rule == "wdep" or c.rule == "hebbian":
        lo, hi = lo - 0.3, hi + 0.3
    r_w = torch.rand(ns, nt, generator=g)
    if c.inf:   # (row 0 and column 0 too: the per-target / per-source forms take them)
        lo[torch.rand(ns, nt, generator=g) < 0.25] = -np.inf
        hi[torch.rand(ns, nt, generator=g) < 0.25] = np.inf
        lo[::3, 0], lo[0, ::4], hi[1::3, 0], hi[0, 1::4] = -np.inf, -np.inf, np.inf, np.inf
    if c.outside and ns > 1 and nt > 1:
        # a per-element lower bound above the upper one (torch.clamp returns wmax) and one equal to it; the per-target /
        # per-source forms take row 0 / column 0, so these elements count only where the bound is full
        lo[ns - 1, nt - 1], hi[ns - 1, nt - 1] = 0.8, 0.5
        lo[ns - 1, nt - 2] = hi[ns - 1, nt - 2] = 0.25
    wmin = _tensor_of(c.lo, lo, g, ns, nt) if c.lo != "scalar" else -0.5
    wmax = _tensor_of(c.hi, hi, g, ns, nt) if c.hi != "scalar" else (np.inf if c.inf else 1.2)
    # the weights start inside the bounds the connection applies (an infinite one read as +-1.5)
    lo_e, hi_e = bcast(wmin, ns, nt).float(), bcast(wmax, ns, nt).float()
    lo_f = torch.where(torch.isfinite(lo_e), lo_e, torch.full((), -1.5))
    hi_f = torch.where(torch.isfinite(hi_e), hi_e, torch.full((), 1.5))
    w = lo_f + (hi_f - lo_f) * (0.15 + 0.7 * r_w)
    if c.outside:
        m = torch.rand(ns, nt, generator=g)
        w = torch.where(m < 0.03, hi_f + 0.4, torch.where(m > 0.97, lo_f - 0.4, w))
    n0, n1 = _rates_scale(c)
    nu_full = [n0 * torch.rand(ns, nt, generator=g), n1 * torch.rand(ns, nt, generator=g)]
    for k in range(2):
        nu_full[k][torch.rand(ns, nt, generator=g) < 0.2] = 0.0
        nu_full[k][0, :] = torch.where(torch.arange(nt) % 5 == 3, torch.zeros(()), nu_full[k][0, :] + 0.2 * (n0, n1)[k])
        nu_full[k][:, 0] = nu_full[k][:, 0] + 0.2 * (n0, n1)[k]   # (so the per-target / per-source rows are not tiny)
    if c.nu == "scalar":
        nu = (f32(n0), f32(n1))
        if c.nu_zero >= 0:
            nu = tuple(0.0 if k == c.nu_zero else nu[k] for k in range(2))
    else:
        nu = [_tensor_of(c.nu, nu_full[k], g, ns, nt) for k in range(2)]
        if c.nu_zero >= 0:
            nu[c.nu_zero] = torch.zeros_like(nu[c.nu_zero])
        nu = tuple(nu)
    # the user weights of the op cases' traces and spikes (the window cases draw them from the run)
    s_src = torch.rand(B, ns, generator=g) < 0.3
    s_tgt = torch.rand(B, nt, generator=g) < 0.08
    if c.events == "all":
        s_tgt[:, 0] = True
    x_src = torch.where(torch.rand(B, ns, generator=g) < 0.25, torch.zeros(()), torch.rand(B, ns, generator=g))
    x_tgt = torch.where(torch.rand(B, nt, generator=g) < 0.25, torch.zeros(()), torch.rand(B, nt, generator=g))
    # the per-neuron population of the <SYN, PN> cases
    pn = draw_pn_population(PnCase("lif", B, 45, T=T, rows=("thresh", "rest", "decay", "trace_decay"), ns=ns), g, ns) if c.pn else None
    if pn is not None:
        pn["x_in"] = x_in   # P hangs off X
    return dict(x_in=x_in, z_in=z_in, w=w.contiguous(), wmin=wmin, wmax=wmax, nu=nu, wd=0.0625 if c.decay else 0.0,
                s_src=s_src, s_tgt=s_tgt, x_src=x_src, x_tgt=x_tgt, pn=pn)


RULE_KW = dict(tc_plus=15.0, tc_minus=25.0, tc_e_trace=10.0)


def _learned_conn(ns_, c: SynCase, d: dict, X, Y):
    L = ns_.learning
    rule = {"postpre": L.PostPre, "wdep": L.WeightDependentPostPre, "hebbian": L.Hebbian, "mstdp": L.MSTDP,
            "mstdpet": L.MSTDPET}[c.rule]
    red = {"sum": torch.sum, "mean": torch.mean}[c.red]
    clone = lambda v: v.clone() if isinstance(v, torch.Tensor) else v
    kw = dict(RULE_KW) if c.rule.startswith("mstdp") else {}
    wmin, wmax = clone(d["wmin"]), clone(d["wmax"])
    tcopy = lambda v: v.t().clone().t()   # a copy with the transposed strides
    if c.lo == "tfull":
        wmin = tcopy(d["wmin"])
    if c.hi == "tfull":
        wmax = tcopy(d["wmax"])
    nu = tuple(clone(v) for v in d["nu"])
    if c.nu == "tfull":
        nu = tuple(tcopy(v) for v in d["nu"])
    conn = ns_.topology.Connection(X, Y, w=d["w"].clone(), update_rule=rule, nu=nu, reduction=red, weight_decay=d["wd"],
                                   wmin=wmin, wmax=wmax, **kw)
    with torch.no_grad():   # (the constructor clamps the user's w, reference topology.py:311-318: weights outside go in afterwards)
        conn.w.copy_(d["w"])
    return conn


def build_syn(ns_, c: SynCase, d: dict):
    """Input X -> LIF Y through the learned Connection, Z -> Y through a large gain (Y spikes one step after Z);
    with ``pn`` also X -> a per-neuron LIF population P through exact static weights.  Returns (net, inputs)."""
    N, T = ns_.nodes, ns_.topology
    net = ns_.Network(dt=1.0, batch_size=c.B, learning=True)
    X, Z = N.Input(c.ns, traces=True), N.Input(c.nt)
    Y = N.LIFNodes(c.nt, traces=True, thresh=Y_THRESH, refrac=0)
    net.add_layer(X, "X"); net.add_layer(Z, "Z"); net.add_layer(Y, "Y")
    net.add_connection(_learned_conn(ns_, c, d, X, Y), "X", "Y")
    net.add_connection(T.Connection(Z, Y, w=Z_GAIN * torch.eye(c.nt)), "Z", "Y")
    from bindsnet_b200.network.monitors import Monitor

    net.add_monitor(Monitor(Y, ["s"], time=c.T), "Ys")
    if c.pn:
        _add_population(ns_, net, d["pn"], X, c.T)
    return net, {"X": d["x_in"], "Z": d["z_in"]}


def run_syn(ns_, c: SynCase, d: dict, device: str = "cpu"):
    """The window (or, ``op``, connection.update() once).  Returns (state, net)."""
    if c.op:
        return run_syn_op(ns_, c, d, device)
    net, inputs = build_syn(ns_, c, d)
    net.force_tier = 1
    if device != "cpu":
        _to_device(net, device)
        inputs = {k: v.to(device) for k, v in inputs.items()}
    kw = dict(reward=c.reward) if c.rule.startswith("mstdp") else {}
    net.run(inputs=inputs, time=c.T, **kw)
    return snapshot(net), net


def run_syn_op(ns_, c: SynCase, d: dict, device: str = "cpu"):
    N = ns_.nodes
    X, Y = N.Input(c.ns, traces=True), N.LIFNodes(c.nt, traces=True)
    for l in (X, Y):
        l.compute_decays(1.0)
        l.set_batch_size(c.B)
    X.s, X.x, Y.s, Y.x = d["s_src"].clone(), d["x_src"].clone(), d["s_tgt"].clone(), d["x_tgt"].clone()
    conn = _learned_conn(ns_, c, d, X, Y)
    if device != "cpu":
        for m in (X, Y, conn):
            m.to(device)
        r = conn.update_rule
        r.nu = r.nu.to(device)
    conn.update(learning=True)
    return {"C/XY/w": conn.w.detach().cpu().clone()}, conn


def _to_device(net, device):
    net.to(device)
    for cn in net.connections.values():
        r = getattr(cn, "update_rule", None)
        if r is not None and isinstance(r.nu, torch.Tensor) and r.nu.dim() > 1:
            r.nu = r.nu.to(device)


def snapshot(net) -> dict:
    """Every layer's s / v / refrac_count / x / theta, every weight, the reward-modulated rules' state, the monitors."""
    out = {}
    for lname, layer in net.layers.items():
        Bz = layer.s.shape[0]
        out[f"L/{lname}/s"] = layer.s.reshape(Bz, -1).to(torch.uint8).cpu()
        for var in ("v", "refrac_count", "x"):
            val = getattr(layer, var, None)
            if isinstance(val, torch.Tensor) and val.numel() > 0:
                out[f"L/{lname}/{var}"] = val.detach().reshape(Bz, -1).float().cpu().clone()
        if isinstance(getattr(layer, "theta", None), torch.Tensor):
            out[f"L/{lname}/theta"] = layer.theta.detach().cpu().clone()
    for (s, t), cn in net.connections.items():
        out[f"C/{s}{t}/w"] = cn.w.detach().cpu().clone()
        for name in ("p_plus", "p_minus", "eligibility_trace", "_spre", "_spost"):
            v = getattr(getattr(cn, "update_rule", None), name, None)
            if isinstance(v, torch.Tensor):
                out[f"R/{s}{t}/{name}"] = v.detach().float().cpu().clone()
    for mname, m in net.monitors.items():
        for var in m.state_vars:
            out[f"M/{mname}/{var}"] = m.get(var).float().cpu().clone()
    return out


def syn_paths(c: SynCase, d: dict, desc=None) -> dict:
    """Which side of each switch of phase3<true> / phase3_mstdp_dense<true> the case takes.  ``desc``: the plan's
    SnnConn of the learned connection (the forms the host chose)."""
    def nu_any(k):
        v = d["nu"][k]
        return bool(v.any()) if isinstance(v, torch.Tensor) else v != 0.0
    pre_on = c.stdp and (nu_any(0) or c.rule == "hebbian")
    post_on = c.stdp and (nu_any(1) or c.rule == "hebbian")
    # Y's spikes of step t are Z's of step t - 1 (the op cases: the given s_tgt)
    if c.op:
        ev = tile_events(d["s_tgt"])
    else:
        ev = max([tile_events(d["z_in"][t - 1].bool()) for t in range(1, c.T)] or [0])
    wmin, wmax = bcast(d["wmin"], c.ns, c.nt), bcast(d["wmax"], c.ns, c.nt)
    has_clamp = bool((wmin != -np.inf).any() or (wmax != np.inf).any())
    out = dict(pre_on=pre_on, post_on=post_on, staged=pre_on and c.B <= XT_STAGED_MAX_B, eager=c.B >= EAGER_B,
               max_events=ev if post_on else 0, overflow=post_on and ev > P3_MAXEV, slots_only=post_on and 0 < ev <= P3_MAXEV,
               row_chunks=not c.op and p3_row_chunks(c.ns, c.nt, EMU_CAP) > 1, warp_loops=c.op and _ceil(c.ns, 32) > GEN_WARPS,
               nt_tail=c.nt % 32 != 0,
               full_decay=c.decay, full_clamp0=has_clamp and not c.decay,
               row_skip=_skips(c, d, has_clamp, group=False), group_skip=_skips(c, d, has_clamp, group=True),
               outside=bool(((d["w"].double() < wmin) | (d["w"].double() > wmax)).any()),
               copied="tfull" in (c.lo, c.hi, c.nu), collapsed=(c.ns == 1 or c.nt == 1),
               mstdp_staged=c.rule.startswith("mstdp") and mstdp_staged(c.B, c.nt))
    if desc is not None:
        from bindsnet_b200 import _abi

        names = {_abi.SNN_SYN_FULL: "FULL", _abi.SNN_SYN_TGT: "TGT", _abi.SNN_SYN_SRC: "SRC", _abi.SNN_SYN_ONE: "ONE"}
        for f in ("wmin", "wmax", "nu0", "nu1"):
            out[f"form_{f}"] = names[getattr(desc, f + "_form")] if getattr(desc, f + "_t") else "scalar"
    return out


def _skips(c: SynCase, d: dict, has_clamp: bool, group: bool) -> bool:
    """phase3's skips of unchanged weights at a step that is not a full pass (no decay, not the clamp pass of step 0):
    a row (``group``: a whole 32-row group of a tile) without a pre-synaptic spike in any sample, in a column (a tile)
    without a post-synaptic event in any sample, is left alone (snn_phases.cuh: the ``tmask`` / ``umask`` tests).
    The op cases run once at t = 0."""
    if not c.stdp or c.decay:
        return False
    steps = [0] if c.op else range(c.T)
    for t in steps:
        if has_clamp and t == 0:
            continue
        if c.op:
            sX, sY = d["s_src"].bool(), d["s_tgt"].bool()
        else:
            sX = d["x_in"][t].bool()
            sY = d["z_in"][t - 1].bool() if t > 0 else torch.zeros(c.B, c.nt, dtype=torch.bool)
        rows, cols = ~sX.any(0), ~sY.any(0)
        if group:
            rg = torch.zeros(_ceil(c.ns, 32) * 32, dtype=torch.bool)
            rg[:c.ns] = rows
            cg = torch.zeros(_ceil(c.nt, 32) * 32, dtype=torch.bool)
            cg[:c.nt] = cols
            cg[c.nt:] = True
            rows_ok = rg.view(-1, 32).clone()
            rows_ok[-1, c.ns % 32 or 32:] = True
            if bool(rows_ok.all(1).any()) and bool(cg.view(-1, 32).all(1).any()):
                return True
        elif bool(rows.any()) and bool(cols.any()):
            return True
    return False


def check_claims(c, paths: dict):
    for k, side in c.claims:
        assert paths[k] == side, f"{c.name}: claims {k} = {side}, the mirror says {paths[k]}"


# ---- float64 restatement of the synapse cases -----------------------------------------------------------------------

def _stdp_step(c: SynCase, d: dict, w, err, sS, xS, sT, xT, gam, wmin, wmax, nu0, nu1, has_clamp):
    """One update of PostPre (learning.py:390-420), WeightDependentPostPre (:626-653) or Hebbian (:1110-1136), then
    the base class (:87-104): decay, clamp with the tensor bounds.  Float64; returns (w', err')."""
    B = sS.shape[0]
    red = (lambda m: m / B) if c.red == "mean" else (lambda m: m)
    g0 = bool(nu0.any()) if not isinstance(nu0, float) else nu0 != 0.0
    g1 = bool(nu1.any()) if not isinstance(nu1, float) else nu1 != 0.0
    terms = w.abs() + err
    if c.rule == "postpre":
        if g0:   # target traces scaled per column before the bmm
            nrow = nu0[0] if nu0.dim() == 2 else nu0
            w = w - red(sS.T @ (xT * nrow))
            terms = terms + red(sS.T @ (xT * nrow).abs())
        if g1:
            nrow = nu1[0] if nu1.dim() == 2 else nu1
            w = w + red(xS.T @ (sT * nrow))
            terms = terms + red(xS.abs().T @ (sT * nrow).abs())
    elif c.rule == "wdep":
        upd = torch.zeros_like(w)
        w0 = w
        if g0:
            upd = upd - nu0 * red(sS.T @ xT) * (w0 - wmin)
            terms = terms + nu0.abs() * red(sS.T @ xT.abs()) * ((w0 - wmin).abs() + err)
        if g1:
            upd = upd + nu1 * red(xS.T @ sT) * (wmax - w0)
            terms = terms + nu1.abs() * red(xS.abs().T @ sT) * ((wmax - w0).abs() + err)
        w = w + upd
    else:   # Hebbian: both rates, ungated
        w = w + nu0 * red(sS.T @ xT)
        w = w + nu1 * red(xS.T @ sT)
        terms = terms + nu0.abs() * red(sS.T @ xT.abs()) + nu1.abs() * red(xS.abs().T @ sT)
    if d["wd"]:
        w = w * (1.0 - d["wd"])
    if has_clamp:
        w = torch.clamp(w, wmin, wmax)
    return w, err + gam * terms


def _f64_rates(c: SynCase, d: dict):
    ns, nt = c.ns, c.nt
    if c.rule == "postpre":   # PostPre's rates broadcast to [1, nt]: keep them per column
        return tuple((bcast(v, 1, nt)[0] if isinstance(v, torch.Tensor) else torch.full((nt,), float(v), dtype=torch.float64))
                     if (isinstance(v, torch.Tensor) and v.any()) or (not isinstance(v, torch.Tensor) and v != 0.0) else 0.0
                     for v in d["nu"])
    return tuple(bcast(v, ns, nt) for v in d["nu"])


def ref_syn(c: SynCase, d: dict, trace_decay: float = 0.0, p_decays: tuple = (), e_decay: float = 0.0):
    """The case in float64.  Windows: Y's raster is Z's one step later (network.py feeds the previous step's spikes),
    the traces follow nodes.py:96-103 with the layers' fp32 decay factor, the rule as restated above.  Returns
    (w, bound, raster of Y [T, B, nt] or None)."""
    f = torch.float64
    ns, nt, B = c.ns, c.nt, c.B
    wmin, wmax = bcast(d["wmin"], ns, nt), bcast(d["wmax"], ns, nt)
    has_clamp = bool((wmin != -np.inf).any() or (wmax != np.inf).any())
    nu0, nu1 = _f64_rates(c, d)
    w, err = d["w"].to(f), torch.zeros(ns, nt, dtype=f)
    if c.op:
        sS, xS, sT, xT = (d[k].to(f) for k in ("s_src", "x_src", "s_tgt", "x_tgt"))
        w, err = _stdp_step(c, d, w, err, sS, xS, sT, xT, gamma(B + 8), wmin, wmax, nu0, nu1, has_clamp)
        return w, err, None
    T = c.T
    xX, xY = torch.zeros(B, ns, dtype=f), torch.zeros(B, nt, dtype=f)
    ys = []
    if c.stdp:
        gam = gamma(B + T + 8)
        for t in range(T):
            sX = d["x_in"][t].bool()
            sY = d["z_in"][t - 1].bool() if t > 0 else torch.zeros(B, nt, dtype=torch.bool)
            xX = torch.where(sX, torch.ones((), dtype=f), xX * trace_decay)
            xY = torch.where(sY, torch.ones((), dtype=f), xY * trace_decay)
            w, err = _stdp_step(c, d, w, err, sX.to(f), xX, sY.to(f), xY, gam, wmin, wmax, nu0, nu1, has_clamp)
            ys.append(sY)
        return w, err, torch.stack(ys)
    # MSTDP (learning.py:1504-1574) / MSTDPET (:2187-2249): the update uses the eligibility of the previous step
    dp, dm = p_decays
    a_plus, a_minus, r = 1.0, -1.0, c.reward
    pp, pm = torch.zeros(B, ns, dtype=f), torch.zeros(B, nt, dtype=f)
    ppa, pma = pp.clone(), pm.clone()      # their absolute-value twins (for the bound)
    sp, st = torch.zeros(B, ns, dtype=f), torch.zeros(B, nt, dtype=f)
    et, eta = torch.zeros(ns, nt, dtype=f), torch.zeros(ns, nt, dtype=f)
    factor = 1.0 - d["wd"] if d["wd"] else 1.0
    red = (lambda m: m.sum(0) / B) if c.red == "mean" else (lambda m: m.sum(0))
    for t in range(T):
        sX = d["x_in"][t].to(f)
        sY = d["z_in"][t - 1].to(f) if t > 0 else torch.zeros(B, nt, dtype=f)
        e = pp.unsqueeze(2) * st.unsqueeze(1) + sp.unsqueeze(2) * pm.unsqueeze(1)          # [B, ns, nt]
        ea = ppa.unsqueeze(2) * st.unsqueeze(1) + sp.unsqueeze(2) * pma.unsqueeze(1)
        w_old = w
        if c.rule == "mstdp":
            w = w + nu0 * red(r * e)
            terms = w_old.abs() + w.abs() + err + nu0.abs() * red(abs(r) * ea)
            err = err + gamma(B + 2 * T + 8) * terms
        else:
            et = et * e_decay + e[0] / RULE_KW["tc_e_trace"]
            eta = eta * e_decay + ea[0] / RULE_KW["tc_e_trace"]
            w = w + ((nu0 * 1.0) * r) * et
            err = err + gamma(5 * T + 10) * (w_old.abs() + w.abs() + err + (nu0 * abs(r)).abs() * eta)
        pp = pp * dp + a_plus * sX
        pm = pm * dm + a_minus * sY
        ppa, pma = ppa * dp + sX, pma * dm + sY
        sp, st = sX, sY
        w = w * factor
        if has_clamp:
            w = torch.clamp(w, wmin, wmax)
        ys.append(sY.bool())
    return w, err, torch.stack(ys)


def ref_syn_two(c: SynCase, d: dict, c2: SynCase, d2: dict, trace_decay: float):
    """Two windows of an STDP case back to back with the same inputs, the bounds and rates of ``d2`` in the second
    one (the traces, Y's last spikes and the bound carry over).  Returns (w, bound)."""
    f = torch.float64
    ns, nt, B, T = c.ns, c.nt, c.B, c.T
    x_in, z_in = torch.cat([d["x_in"], d["x_in"]]), torch.cat([d["z_in"], d["z_in"]])
    w, err = d["w"].to(f), torch.zeros(ns, nt, dtype=f)
    xX, xY = torch.zeros(B, ns, dtype=f), torch.zeros(B, nt, dtype=f)
    gam = gamma(B + 2 * T + 8)
    for t in range(2 * T):
        cc, dd = (c, d) if t < T else (c2, d2)
        wmin, wmax = bcast(dd["wmin"], ns, nt), bcast(dd["wmax"], ns, nt)
        has_clamp = bool((wmin != -np.inf).any() or (wmax != np.inf).any())
        nu0, nu1 = _f64_rates(cc, dd)
        sX = x_in[t].bool()
        sY = z_in[t - 1].bool() if t > 0 else torch.zeros(B, nt, dtype=torch.bool)
        xX = torch.where(sX, torch.ones((), dtype=f), xX * trace_decay)
        xY = torch.where(sY, torch.ones((), dtype=f), xY * trace_decay)
        w, err = _stdp_step(cc, dd, w, err, sX.to(f), xX, sY.to(f), xY, gam, wmin, wmax, nu0, nu1, has_clamp)
    return w, err


def rule_decays(net):
    """(trace decay of X, (p_plus, p_minus) decays, e_trace decay) as the layers / rule hold them in fp32."""
    cn = net.connections[("X", "Y")]
    r = cn.update_rule
    td = float(net.layers["X"].trace_decay)
    if not hasattr(r, "tc_plus"):
        return td, (), 0.0
    pd = (float(torch.exp(-1.0 / r.tc_plus)), float(torch.exp(-1.0 / r.tc_minus)))
    ed = float(torch.exp(-1.0 / r.tc_e_trace)) if hasattr(r, "tc_e_trace") else 0.0
    return td, pd, ed


# ---- per-neuron parameter cases -------------------------------------------------------------------------------------

@dataclass(frozen=True)
class PnCase:
    kind: str                 # lif / alif / dc (DiehlAndCookNodes with one_spike)
    B: int
    n: int
    T: int = 8
    rows: tuple = PN_ROWS     # which parameters are per-neuron tensors
    one_step: bool = False
    learning: bool = True     # the network's learning flag (theta adapts only while learning)
    windows: int = 1          # consecutive windows without a reset
    additive: bool = True     # traces_additive (a per-neuron trace_scale needs it)
    lbound: bool = False      # a scalar lower bound on v, reached by strongly negative inputs
    conv: bool = False        # Input [2, H, W] -> Conv2dConnection -> a [C, H, W] population with a [C, 1, 1] threshold
    ns: int = 40
    seed: int = 0
    claims: tuple = ()
    gpu: tuple = ()           # (B, T) on the GPU

    @property
    def name(self) -> str:
        rows = "all" if set(self.rows) == set(PN_ROWS) or (self.kind == "lif" and set(self.rows) == set(lif_rows())) \
            else "+".join(self.rows) if self.rows else "none"
        extra = "".join(["_onestep" if self.one_step else "", "_nolearn" if not self.learning else "",
                         f"_w{self.windows}" if self.windows > 1 else "", "_add" if self.additive else "",
                         "_lbound" if self.lbound else "", "_conv" if self.conv else "", f"_s{self.seed}" if self.seed else ""])
        return f"{self.kind}_b{self.B}_n{self.n}_T{self.T}_{rows}{extra}"

    def at_gpu_size(self) -> "PnCase":
        return replace(self, B=self.gpu[0], T=self.gpu[1]) if self.gpu else self

    @property
    def theta(self) -> bool:
        return self.kind in ("alif", "dc")


def lif_rows():
    return ("thresh", "rest", "decay", "trace_decay", "trace_scale")


def _pn_cases():
    P = PnCase
    cases = []
    # every row alone (a row-index mix-up shows), on the population that has it
    for i, r in enumerate(PN_ROWS):
        kind = "alif" if r.startswith("theta") else "lif"
        cases.append(P(kind, 3, 45, rows=(r,), additive=r == "trace_scale", seed={"decay": 10, "theta_decay": 10}.get(r, i), claims=((f"row_{r}", True),)))
    cases += [
        P("lif", 4, 45, rows=lif_rows(), additive=True, claims=(("n_tail", True),)),
        P("alif", 4, 64, additive=True, claims=(("n_tail", False),)),
        P("dc", 3, 45, rows=("thresh", "decay", "theta_plus", "trace_decay"), claims=(("one_spike", True),)),
        P("dc", 4, 33, additive=True, claims=(("one_spike", True),)),
        P("dc", 5, 45, rows=("trace_decay", "trace_scale"), additive=True, claims=(("one_spike", True),)),
        P("dc", 70, 45, T=4, additive=True, claims=(("chunks", True), ("one_spike", True)), gpu=(200, 6)),
        P("lif", 100, 45, T=4, rows=lif_rows(), additive=True, claims=(("chunks", True),), gpu=(300, 6)),
        P("alif", 100, 45, T=4, claims=(("chunks", True),)),
        P("lif", 3, 45, rows=lif_rows(), additive=True, one_step=True, claims=(("one_step", True),)),
        P("dc", 3, 45, additive=True, one_step=True, claims=(("one_step", True), ("one_spike", True))),
        P("alif", 3, 45, one_step=True, windows=2, claims=(("one_step", True),)),
        P("alif", 3, 45, learning=False, claims=(("theta_learning", False),)),
        P("dc", 3, 45, learning=False, additive=True),
        P("alif", 3, 45, T=1, windows=5, claims=(("T1", True),)),
        P("dc", 2, 45, T=1, windows=3, additive=True, claims=(("T1", True), ("windows", 3))),
        P("alif", 3, 45, windows=2, claims=(("windows", 2),)),
        P("lif", 3, 45, rows=("thresh", "rest", "decay"), windows=2, lbound=True),
        P("lif", 3, 147, rows=("thresh",), conv=True, claims=(("per_channel", True), ("n_tail", True))),
        P("lif", 2, 147, rows=("thresh", "decay"), conv=True, windows=2),
    ]
    return cases


PN_CASES = _pn_cases()


def _pn_values(kind: str, n: int, g: torch.Generator, rows, additive: bool, conv: bool):
    """The population's parameters: per-neuron tensors for ``rows``, the scalars otherwise."""
    vec = lambda lo, hi: (lo + (hi - lo) * torch.rand(n, generator=g)).view(*([3, 7, 7] if conv else [n]))
    v = dict(thresh=-56.0 if kind == "lif" else -55.0, rest=-65.0, tc_decay=30.0, theta_plus=0.25, tc_theta_decay=60.0,
             tc_trace=20.0, trace_scale=0.75 if additive else 1.0)
    for r in rows:
        if r == "thresh":
            v["thresh"] = torch.tensor([-60.0, -57.0, -54.5]).view(3, 1, 1) if conv else vec(-59.0, -53.0)
        elif r == "rest":
            v["rest"] = vec(-68.0, -62.0)
        elif r == "decay":
            v["tc_decay"] = vec(8.0, 120.0)
        elif r == "theta_plus":
            v["theta_plus"] = vec(0.05, 0.8)
        elif r == "theta_decay":
            v["tc_theta_decay"] = vec(5.0, 400.0)
        elif r == "trace_decay":
            v["tc_trace"] = vec(3.0, 40.0)
        elif r == "trace_scale":
            v["trace_scale"] = vec(0.3, 1.7)
    return v


def draw_pn_population(c: PnCase, g: torch.Generator, ns: int) -> dict:
    """Parameters, static input weights (multiples of 1/8: every input sum is exact in fp32) and input spikes."""
    vals = _pn_values(c.kind, c.n, g, c.rows, c.additive, c.conv)
    if c.conv:
        w = torch.randint(-2, 7, (3, 2, 3, 3), generator=g).float() / 8.0
        x_in = (torch.rand(c.windows * c.T, c.B, 2, 7, 7, generator=g) < 0.35).to(torch.uint8)
    else:
        k = torch.randint(-4, 13, (ns, c.n), generator=g).float()
        if c.lbound:   # a third of the neurons get strongly inhibitory inputs
            k[:, ::3] = -torch.randint(6, 16, (ns, len(range(0, c.n, 3))), generator=g).float()
        w = k / 8.0
        x_in = (torch.rand(c.windows * c.T, c.B, ns, generator=g) < 0.22).to(torch.uint8)
    return dict(case=c, vals=vals, w=w, x_in=x_in)


def draw_pn(c: PnCase) -> dict:
    g = torch.Generator().manual_seed(4099 + 7919 * c.seed + 131 * c.B + c.n + 3 * c.T + len(c.rows) + 1000 * c.windows)
    return draw_pn_population(c, g, c.ns)


def _add_population(ns_, net, p: dict, X, T):
    c, v = p["case"], p["vals"]
    N = ns_.nodes
    kw = dict(traces=True, traces_additive=c.additive, tc_trace=v["tc_trace"], trace_scale=v["trace_scale"], refrac=3,
              reset=-64.0, thresh=v["thresh"], rest=v["rest"], tc_decay=v["tc_decay"])
    if c.conv:
        kw["shape"] = [3, 7, 7]
    else:
        kw["n"] = c.n
    if c.kind == "lif":
        P = N.LIFNodes(lbound=-70.0 if c.lbound else None, **kw)
    else:
        kw.update(theta_plus=v["theta_plus"], tc_theta_decay=v["tc_theta_decay"])
        P = (N.AdaptiveLIFNodes if c.kind == "alif" else N.DiehlAndCookNodes)(**kw, **({} if c.kind == "alif" else {"one_spike": True}))
    net.add_layer(P, "P")
    if c.conv:
        conn = ns_.topology.Conv2dConnection(X, P, kernel_size=3, stride=1, padding=1, w=p["w"].clone())
    else:
        conn = ns_.topology.Connection(X, P, w=p["w"].clone())
    net.add_connection(conn, X_name(net, X), "P")
    from bindsnet_b200.network.monitors import Monitor

    net.add_monitor(Monitor(P, ["s", "v"], time=T), "Pm")
    return P


def X_name(net, X):
    return next(k for k, l in net.layers.items() if l is X)


def build_pn(ns_, c: PnCase, d: dict):
    net = ns_.Network(dt=1.0, batch_size=c.B, learning=c.learning)
    X = ns_.nodes.Input(shape=[2, 7, 7]) if c.conv else ns_.nodes.Input(c.ns)
    net.add_layer(X, "X")
    _add_population(ns_, net, d, X, c.T)
    return net


def run_pn(ns_, c: PnCase, d: dict, device: str = "cpu"):
    """``windows`` windows of T steps without a reset; returns (per-window snapshots, net)."""
    net = build_pn(ns_, c, d)
    net.force_tier = 1
    if device != "cpu":
        net.to(device)
    torch.manual_seed(5)   # (the one_spike tie-break seed Network.run draws)
    outs = []
    for k in range(c.windows):
        x = d["x_in"][k * c.T:(k + 1) * c.T]
        net.run(inputs={"X": x.to(device)}, time=c.T, one_step=c.one_step)
        outs.append(snapshot(net))
    return outs, net


def pn_paths(c: PnCase, net=None) -> dict:
    n_x = 98 if c.conv else c.ns
    items = _ceil(n_x, 32) + _ceil(c.n, 32)
    out = {f"row_{r}": r in c.rows and (c.kind != "lif" or not r.startswith("theta")) for r in PN_ROWS}
    out.update(n_tail=c.n % 32 != 0, chunks=sample_chunks(c.B, items, EMU_CAP) > 1, one_step=c.one_step,
               one_spike=c.kind == "dc", theta_learning=c.theta and c.learning, T1=c.T == 1, windows=c.windows,
               per_channel=c.conv, lbound=c.lbound)
    if net is not None:   # the rows the host put into the layer's block
        from bindsnet_b200 import _abi

        d = _abi.SnnLayer()
        P = net.layers["P"]
        P._fill_desc(d)
        mask = int(d.pn_mask) if d.kind & _abi.SNN_NODE_PN else 0
        out["mask_rows"] = tuple(r for i, r in enumerate(PN_ROWS) if (mask >> i) & 1)
    return out


# ---- float64 restatement of the neuron cases ------------------------------------------------------------------------

def _exp64(tc):
    tc = tc if isinstance(tc, torch.Tensor) else torch.tensor(float(tc))
    return torch.exp(-1.0 / tc.to(torch.float32).to(torch.float64))


def check_decay_factors(P):
    """|decay_32 - decay_64| <= 3u decay_64 for every fp32 factor the population holds (the bound's premise)."""
    pairs = [(P.decay, P.tc_decay), (P.trace_decay, P.tc_trace)]
    if hasattr(P, "theta_decay"):
        pairs.append((P.theta_decay, P.tc_theta_decay))
    for d32, tc in pairs:
        d64 = _exp64(tc.cpu())
        rel = ((d32.cpu().to(torch.float64) - d64).abs() / d64).max()
        assert float(rel) <= DECAY_REL, f"an fp32 decay factor is {float(rel) / U32:.2f} u from exp(-dt / tc)"


def _flat(v, shape, n):
    """A parameter as float64 [n] (per-neuron tensors broadcast to the layer's shape)."""
    if isinstance(v, torch.Tensor) and v.numel() > 1:
        return v.to(torch.float64).expand(*shape).reshape(-1).clone()
    return torch.full((n,), float(v), dtype=torch.float64)


def pn_input(c: PnCase, d: dict, s_x: torch.Tensor) -> torch.Tensor:
    """The population's input for the source spikes ``s_x`` [B, *X.shape] (topology.py Connection / Conv2dConnection
    .compute), float64; exact in fp32 (multiples of 1/8)."""
    sx = s_x.to(torch.float64)
    if c.conv:
        import torch.nn.functional as F

        return F.conv2d(sx, d["w"].to(torch.float64), None, padding=1).reshape(sx.shape[0], -1)
    return sx.reshape(sx.shape[0], -1) @ d["w"].to(torch.float64)


def ref_pn(c: PnCase, d: dict, outs: list, P) -> dict:
    """The population in float64, teacher-forced with the oracle's spikes (``outs``: per-window snapshots, whose
    monitor ``Pm`` holds s and v of every step).  nodes.py:500-529 (LIFNodes), :921-946 (AdaptiveLIFNodes), :1069-1110
    (DiehlAndCookNodes), :96-103 (traces).  Returns the float64 states, their bounds, and the margin and raster
    checks: {"v": [windows][T, B, n], "v_err", "x", "x_err", "theta", "theta_err", "rc", "margin_ok", "raster_ok"}."""
    f = torch.float64
    n, B, shape = c.n, c.B, list(P.shape)
    v = d["vals"]
    thresh, rest = _flat(v["thresh"], shape, n), _flat(v["rest"], shape, n)
    dec = _flat(_exp64(v["tc_decay"] if isinstance(v["tc_decay"], torch.Tensor) else torch.tensor(v["tc_decay"])), shape, n)
    tdec = _flat(_exp64(v["tc_trace"] if isinstance(v["tc_trace"], torch.Tensor) else torch.tensor(v["tc_trace"])), shape, n)
    scale = _flat(torch.as_tensor(v["trace_scale"], dtype=torch.float32), shape, n)
    tplus = _flat(torch.as_tensor(v["theta_plus"], dtype=torch.float32), shape, n)
    thdec = _flat(_exp64(v["tc_theta_decay"] if isinstance(v["tc_theta_decay"], torch.Tensor) else torch.tensor(v["tc_theta_decay"])), shape, n)
    reset, refrac, lb = -64.0, 3.0, (-70.0 if c.lbound else None)
    learning = c.theta and c.learning
    V = torch.full((B, n), 0.0, dtype=f) + rest
    E = torch.zeros(B, n, dtype=f)
    RC = torch.zeros(B, n, dtype=f)
    X, EX = torch.zeros(B, n, dtype=f), torch.zeros(B, n, dtype=f)
    TH, ETH = torch.zeros(n, dtype=f), torch.zeros(n, dtype=f)
    s_prev_x = torch.zeros(B, *(([2, 7, 7]) if c.conv else [c.ns]), dtype=torch.uint8)
    g5, g3 = gamma(5), gamma(3)
    res = dict(v=[], v_err=[], x=[], x_err=[], theta=[], theta_err=[], rc=[], margin_ok=True, raster_ok=True, min_margin=np.inf)
    for k in range(c.windows):
        s_oracle = outs[k]["M/Pm/s"].reshape(c.T, B, n).bool()
        vs, es = [], []
        for t in range(c.T):
            xin_s = d["x_in"][k * c.T + t]
            I = pn_input(c, d, xin_s if c.one_step else s_prev_x)
            s_prev_x = xin_s
            a = dec * (V - rest)
            Vn = a + rest
            thr = thresh
            if c.kind != "lif" and learning:
                tnew = TH * thdec
                ETH = thdec * (1 + DECAY_REL) * ETH + (DECAY_REL + gamma(1)) * tnew.abs()
                TH = tnew
            gate = (RC <= 0).to(f)
            Vn = Vn + gate * I
            E = dec * (1 + DECAY_REL) * E + g5 * (a.abs() + rest.abs() + I.abs() + Vn.abs()) + DECAY_REL * a.abs()
            RC = RC - 1.0
            if c.kind == "lif":
                thr_v, thr_err = thresh.expand(B, n), torch.zeros(B, n, dtype=f)
            else:
                thr_v = (thresh + TH).expand(B, n)
                thr_err = (ETH + U32 * (thresh + TH).abs()).expand(B, n)
            gap = (Vn - thr_v).abs() - (E + thr_err)
            res["min_margin"] = min(res["min_margin"], float(gap.min()))
            if bool((gap <= 0).any()):
                res["margin_ok"] = False
            cand = Vn >= thr_v
            if c.kind == "dc":   # one_spike: the oracle's winners are among the candidates, one per sample with any
                fin = s_oracle[t]
                if not (bool((fin & ~cand).any()) is False and torch.equal(fin.sum(1), cand.any(1).to(torch.int64))):
                    res["raster_ok"] = False
            else:
                fin = cand
                if not torch.equal(cand, s_oracle[t]):
                    res["raster_ok"] = False
            RC = torch.where(cand, torch.full((), refrac, dtype=f), RC)
            Vn = torch.where(cand, torch.full((), reset, dtype=f), Vn)
            E = torch.where(cand, torch.zeros((), dtype=f), E)
            if lb is not None:
                E = torch.where(Vn < lb, torch.zeros((), dtype=f), E)
                Vn = torch.where(Vn < lb, torch.full((), lb, dtype=f), Vn)
            if c.kind != "lif" and learning:
                cnt = cand.to(f).sum(0)
                tnew = TH + tplus * cnt
                ETH = ETH + gamma(2) * ((tplus * cnt).abs() + tnew.abs())
                TH = tnew
            # traces (nodes.py:96-103) with the final spikes
            xd = X * tdec
            if c.additive:
                Xn = xd + scale * fin.to(f)
                EX = tdec * (1 + DECAY_REL) * EX + (DECAY_REL + g3) * (xd.abs() + scale.abs() + Xn.abs())
            else:
                Xn = torch.where(fin, scale.expand(B, n), xd)
                EX = torch.where(fin, torch.zeros((), dtype=f), tdec * (1 + DECAY_REL) * EX + (DECAY_REL + g3) * xd.abs())
            X = Xn
            V = Vn
            vs.append(V.clone()); es.append(E.clone())
        res["v"].append(torch.stack(vs)); res["v_err"].append(torch.stack(es))
        res["x"].append(X.clone()); res["x_err"].append(EX.clone())
        res["theta"].append(TH.clone()); res["theta_err"].append(ETH.clone()); res["rc"].append(RC.clone())
    return res
