"""Edge cases of the generic kernel's sparse instantiation (``snn_generic_window<2, true, ...>``: ``sparse_prepass``,
``phase_sparse`` and ``decay_sparse`` in csrc/snn_phases.cuh, ``sparse_block_width`` in csrc/snn_common.cuh, the unit
layout of ``plan_units`` in csrc/snn_generic.cu) and of its single operators (``sparse_compute_kernel`` and the NoOp
branch of ``snn_b200_conn_update`` in csrc/snn_ops.cu), with plain float64 restatements of the reference's formulas and
Python mirrors of the kernels' path conditions.  Shared by tests/test_sparse_edges.py (CPU: the oracle against float64,
the emulated kernel against the oracle) and tests/test_gpu_sparse_edges.py (the CUDA library).  No test functions here.

The restatements are written from the reference (topology.py, network.py, nodes.py, learning.py); the oracle that runs
the cases is tests/sparse_oracle.c.

Error bounds
------------
u = 2**-24 and gamma_k = k u / (1 - k u) as in tests/kernel_edges.py.

Input.  ``SparseConnection.compute`` is ``s.float() @ w + b`` (topology.py:332-346, :2009-2017): for sample b and target
j the stored w_ij of the spiking i plus b_j.  The target's input adds every connection into it in insertion order,
starting from zeros (network.py:211-250).  So the input of (b, j) is a sum of k stored entries gathered, the dense
connections' weights of the spiking sources and the biases; summed through at most k + 2 roundings in any order it is
within gamma_{k+2} times the sum of the absolute values of its terms (Higham, Lemma 3.1 and §3.1), k counting every
term.  A source that did not spike adds no term, as in the kernels' gathers: an infinite stored value of a silent source
does not turn the sum into NaN as the 0 * inf of a dense product would.

Decay.  learning.NoOp scales w by ``1 - weight_decay`` when that is non-zero (learning.py:85-94), so 1.0 leaves w alone
and 2.0 flips its sign every step.  The kernel holds the factor as fp32 and rounds ``w * factor`` once per step: after t
steps a stored value is within gamma_t |w f^t| of the float64 product of the fp32 factor (an exact factor of -1 or 1
leaves the value exact).  A gathered entry then carries (1 + gamma_t), and the input's bound becomes gamma_{k+2+t}.

Neurons.  The input carries the bound e_x above; it enters the voltage through one addition, whose rounding is already
counted, so each voltage step adds e_x to the bound of the step with an exact input:
* LIFNodes (nodes.py:500-529): the step bound tests/param_edges.py derives and ``ref_pn`` applies
  (``lif_step_err`` here) plus e_x.
* IFNodes (nodes.py:371-395): ``v' = fl(v + gate x)``, so e' = e + u |v'| + e_x.
* CurrentLIFNodes (nodes.py:762-789): ``i' = fl(fl(i_decay i) + x)`` with the fp32 factor within 3u of the float64 one
  (param_edges.DECAY_REL): e_i' = i_decay (1 + gamma_5) e_i + gamma_5 (|i_decay i| + |i'|) + e_x, and the voltage step
  is the LIF one with input i' carrying e_i'.
The threshold compare is exact.  The voltages are teacher-forced with the oracle's spikes: every neuron-step's float64
voltage must lie farther than its bound from the threshold, and the float64 raster must equal the oracle's.  A
non-finite float64 voltage (the inf case) is compared by class, not by value, and needs no margin.
"""
from __future__ import annotations

from dataclasses import dataclass, replace

import numpy as np
import torch

from kernel_edges import f32, gamma
from param_edges import DECAY_REL

U32 = 2.0 ** -24
GEN_WARPS = 8            # SNN_GEN_WARPS: samples per gather unit
GROUP = 1024             # sources compacted per pass of phase_sparse's w0 loop (32 words)
UNITS_MIN = 200          # sparse_block_width narrows the blocks until there are about this many units
OFF_CAP = 16 * 2 ** 20   # ... and never beyond this many bytes of offset table (or 16 nnz bytes)
OP_GRID_Y = 64           # snn_b200_conn_compute caps grid.y
OP_UPDATE_BLOCKS = 1184  # snn_b200_conn_update's scale_kernel: at most 1184 CTAs of 256 threads, 1024 values per CTA
THRESH = dict(lif=-58.0, clif=-58.0, iff=-60.0)


def _ceil(a, b):
    return (a + b - 1) // b


# ---- path mirrors -------------------------------------------------------------------------------------------------

def block_width(ns: int, nt: int, B: int, nnz: int) -> tuple:
    """sparse_block_width (snn_common.cuh) and why it stopped: "floor" (128), "units" (enough units), "cap" (the next
    halving would outgrow the offset table)."""
    cap = max(16.0 * nnz, float(OFF_CAP))
    bw = 1024
    while True:
        if bw <= 128:
            return bw, "floor"
        if _ceil(nt, bw) * _ceil(B, GEN_WARPS) >= UNITS_MIN:
            return bw, "units"
        if 4.0 * ns * (_ceil(nt, bw // 2) + 1) > cap:
            return bw, "cap"
        bw //= 2


# ---- cases --------------------------------------------------------------------------------------------------------

@dataclass(frozen=True)
class SparseCase:
    ns: int
    nt: int
    B: int
    T: int = 4
    kind: str = "lif"         # the target Y: lif / iff / clif
    values: str = "mixed"     # mixed signs / "zeros": explicit stored zeros too / "inf": +-inf entries
    wd: float = -1.0          # learning.NoOp(weight_decay=wd) on the sparse connections; < 0: no rule
    density: float = 0.08
    bias: bool = True
    dense: bool = False       # a dense Connection Z -> Y after the sparse one (insertion order)
    rows: bool = False        # engineered rows: 1 / 32 / 33 / 70 entries in block 0, a row only in a later block,
                              # columns 0, j0 + bw - 1 and nt - 1
    two: int = 0              # a second SparseConnection X -> Y2 (IF, this many targets): another width, sp[1].first > 0
    rec: bool = False         # a recurrent SparseConnection Y -> Y
    order: str = "sync"       # sync / before (one-step, X before Y) / after (one-step, Y before X) / rec (one-step, Y -> Y)
    windows: int = 1
    nnz0: bool = False        # X -> Y stores nothing
    seed: int = 0
    claims: tuple = ()
    gpu: tuple = ()           # (B, T) on the GPU where the CPU file runs a smaller case

    @property
    def name(self) -> str:
        extra = "".join([f"_wd{self.wd:g}" if self.wd >= 0 else "", "_nob" if not self.bias else "", "_dense" if self.dense else "",
                         "_rows" if self.rows else "", f"_two{self.two}" if self.two else "", "_rec" if self.rec else "",
                         f"_{self.order}" if self.order != "sync" else "", f"_w{self.windows}" if self.windows > 1 else "",
                         "_nnz0" if self.nnz0 else "", f"_{self.values}" if self.values != "mixed" else "",
                         f"_s{self.seed}" if self.seed else ""])
        return f"{self.kind}_{self.ns}x{self.nt}_b{self.B}_T{self.T}{extra}"

    @property
    def one_step(self) -> bool:
        return self.order != "sync"

    def at_gpu_size(self) -> "SparseCase":
        return replace(self, B=self.gpu[0], T=self.gpu[1]) if self.gpu else self


def _cases():
    S = SparseCase
    return [
        # the block widths: 1024 and 512 stop on the unit count, 256 on the offset-table cap, 128 at the floor
        S(40, 8192, 200, T=2, kind="iff", rows=True, density=0.02, two=300, wd=0.1,
          claims=(("bw", 1024), ("stop", "units"), ("partial", False), ("two_widths", True), ("b_tail", 0))),
        S(40, 4000, 200, T=2, kind="iff", density=0.02, claims=(("bw", 512), ("stop", "units"), ("partial", True))),
        S(40_000, 16384, 1, T=3, kind="iff", density=0.00004, rows=True, wd=2.0, gpu=(8, 3),
          claims=(("bw", 256), ("stop", "cap"), ("words_gt32", True))),
        S(70, 300, 3, T=5, kind="lif", wd=0.1, dense=True, claims=(("bw", 128), ("stop", "floor"), ("partial", True))),
        # rows with 0 / 1 / 32 / 33 / 70 entries in a block, a row whose entries lie in a later block, the edge columns
        S(100, 300, 9, T=5, kind="lif", rows=True, dense=True, wd=0.1, claims=(("b_tail", 1), ("late_row", True))),
        S(100, 256, 16, T=4, kind="clif", rows=True, wd=1.0, claims=(("partial", False), ("b_tail", 0))),
        # source widths around a word and a 1024-source group
        S(1, 40, 1, T=6, kind="clif", density=0.6, wd=0.0, claims=(("b_tail", 1),)),
        S(31, 33, 7, T=5, kind="iff", values="zeros", density=0.3, wd=0.1, claims=(("b_tail", 7),)),
        S(32, 256, 8, T=4, kind="lif", density=0.3, wd=1.0, claims=(("b_tail", 0), ("nb_gt1", True))),
        S(33, 50, 16, T=4, kind="lif", density=0.3, order="before", claims=(("cur", True),)),
        S(1024, 200, 5, T=5, kind="lif", density=0.02, claims=(("words_gt32", False), ("all_group", True))),
        S(1025, 130, 5, T=4, kind="iff", density=0.02, order="after", wd=0.1,
          claims=(("words_gt32", True), ("anyf_skip", True), ("prev_one_step", True))),
        S(3000, 150, 4, T=5, kind="clif", density=0.01, wd=2.0, claims=(("anyf_skip", True), ("step0_slot2", True))),
        S(1500, 140, 3, T=4, kind="lif", density=0.01, order="before", claims=(("cur", True), ("anyf_skip", True))),
        # nnz = 0, +-inf, recurrent (sync and one-step), two windows
        S(50, 70, 2, T=4, kind="lif", nnz0=True, dense=True, claims=(("nnz0", True),)),
        S(60, 40, 3, T=4, kind="iff", values="inf", density=0.2, bias=False),
        S(70, 100, 3, T=5, kind="lif", rec=True, wd=0.1, density=0.1),
        S(70, 100, 3, T=5, kind="lif", rec=True, order="rec", density=0.1, claims=(("prev_one_step", True),)),
        S(1100, 90, 2, T=3, kind="clif", density=0.02, rec=True, order="before", windows=2, wd=0.1,
          claims=(("cur", True), ("prev_one_step", True), ("windows", 2))),
        S(70, 300, 9, T=3, kind="lif", rows=True, wd=2.0, windows=2, claims=(("windows", 2),)),
    ]


CASES = _cases()


# ---- drawing ------------------------------------------------------------------------------------------------------

COUNTS = ("rand", 0, 1, 8, 9, 32, 33, "all")   # spiking sources of group 0 at (t, b): cycled over t + b


def _pattern(ns, nt, density, g) -> torch.Tensor:
    """[2, nnz] int64 positions of a random pattern of about the given density, row-major."""
    if ns * nt <= 20_000_000:
        return (torch.rand(ns, nt, generator=g) < density).nonzero().T.contiguous()
    flat = torch.unique(torch.randint(0, ns * nt, (int(density * ns * nt),), generator=g, dtype=torch.int64))
    return torch.stack([flat // nt, flat % nt])


def _set_row(idx: torch.Tensor, i: int, cols) -> torch.Tensor:
    cols = torch.as_tensor(cols, dtype=torch.int64).unique()
    keep = idx[:, idx[0] != i]
    return torch.cat([keep, torch.stack([torch.full_like(cols, i), cols])], 1)


def _rows(idx: torch.Tensor, ns: int, nt: int, bw: int, g) -> tuple:
    """Engineered rows (where the source is wide enough): entries 1 / 32 / 33 / 70 in block 0, one row only in the last
    block, columns 0, bw - 1 (the last column of block 0), j0 + bw - 1 of the last full block and nt - 1."""
    rows = []
    want = [n for n in (1, 32, 33, 70) if n <= min(bw, nt)]
    for k, n in enumerate(want):
        i = (7 * k + 3) % ns
        idx = _set_row(idx, i, torch.randperm(min(bw, nt), generator=g)[:n])
        rows.append(i)
    nb = _ceil(nt, bw)
    if nb > 1:
        i = (7 * len(want) + 3) % ns
        j0 = (nb - 1) * bw
        idx = _set_row(idx, i, j0 + torch.randperm(nt - j0, generator=g)[:min(5, nt - j0)])
        rows.append(i)
    i = (7 * len(rows) + 3) % ns
    edge = [0, min(bw, nt) - 1, nt - 1] + ([(nt // bw) * bw - 1] if nt >= 2 * bw else [])
    idx = _set_row(idx, i, torch.cat([idx[1, idx[0] == i], torch.tensor(edge)]))
    rows.append(i)
    return idx, rows


def _values(idx: torch.Tensor, shape, values, g, scale):
    idx = torch.sparse_coo_tensor(idx, torch.zeros(idx.shape[1]), shape).coalesce().indices()
    k = idx.shape[1]
    v = scale * (0.5 + 2.0 * torch.rand(k, generator=g)) * torch.where(torch.rand(k, generator=g) < 0.6, 1.0, -1.0)
    if values == "zeros" and k:
        z = torch.rand(k, generator=g) < 0.3
        v = torch.where(z, torch.where(torch.rand(k, generator=g) < 0.5, 0.0, -0.0), v)
    if values == "inf" and k > 3:
        # +inf and -inf in one column (NaN where both rows spike), +inf alone in another
        cols = idx[1]
        j = int(cols[0])
        same = (cols == j).nonzero().flatten()
        v[same[0]] = np.inf
        if same.numel() > 1:
            v[same[1]] = -np.inf
        other = (cols != j).nonzero().flatten()
        v[other[0]] = np.inf
    return torch.sparse_coo_tensor(idx, v, tuple(shape)).coalesce()


def _spikes(T, B, n, g, p, engineered=()):
    """[T, B, n] spikes: group 0 (the first 1024 sources) has COUNTS[(t + b) % 8] spiking sources; a count of 0 leaves
    the whole sample silent; "rand" switches the engineered rows on."""
    x = (torch.rand(T, B, n, generator=g) < p)
    g0 = min(n, GROUP)
    for t in range(T):
        for b in range(B):
            c = COUNTS[(t + b) % len(COUNTS)]
            if c == "rand":
                for i in engineered:
                    x[t, b, i] = True
                continue
            x[t, b, :g0] = False
            if c == "all":
                x[t, b, :g0] = True
            elif c == 0:
                x[t, b, :] = False
            else:
                x[t, b, torch.randperm(g0, generator=g)[:min(c, g0)]] = True
    return x.to(torch.uint8)


def draw(c: SparseCase) -> dict:
    g = torch.Generator().manual_seed(3301 + 7919 * c.seed + 131 * c.B + 17 * c.ns + c.nt + 3 * c.T)
    steps = c.T * c.windows
    idx = _pattern(c.ns, c.nt, 0.0 if c.nnz0 else c.density, g)
    # (the width depends on nnz only beyond 2**20 entries: the engineered rows follow the final width)
    bw, _ = block_width(c.ns, c.nt, c.B, idx.shape[1])
    rows = []
    if c.rows:
        idx, rows = _rows(idx, c.ns, c.nt, bw, g)
    scale = 3.0 if c.kind != "iff" else 2.0
    d = dict(w=_values(idx, (c.ns, c.nt), c.values, g, scale), rows=rows)
    d["b"] = 0.5 * torch.rand(c.nt, generator=g) - 0.1 if c.bias else None
    d["x"] = _spikes(steps, c.B, c.ns, g, 0.2 if c.ns < 2000 else 0.05, rows)
    if c.dense:
        d["wz"] = torch.randn(20, c.nt, generator=g) * 1.5
        d["z"] = (torch.rand(steps, c.B, 20, generator=g) < 0.2).to(torch.uint8)
    if c.two:
        d["w2"] = _values(_pattern(c.ns, c.two, 0.3, g), (c.ns, c.two), "mixed", g, 4.0)
    if c.rec:
        d["wr"] = _values(_pattern(c.nt, c.nt, 0.1, g), (c.nt, c.nt), "mixed", g, 1.5)
    return d


# ---- the network --------------------------------------------------------------------------------------------------

def _target(N, kind, n):
    kw = dict(traces=True, reset=-64.0, refrac=2)
    if kind == "iff":
        return N.IFNodes(n, thresh=THRESH["iff"], **kw)
    if kind == "lif":
        return N.LIFNodes(n, thresh=THRESH["lif"], rest=-65.0, tc_decay=20.0, **kw)
    return N.CurrentLIFNodes(n, thresh=THRESH["clif"], rest=-65.0, tc_decay=20.0, tc_i_decay=2.0, **kw)


def build(ns_, c: SparseCase, d: dict):
    """X -> Y (SparseConnection), then Z -> Y (dense), X -> Y2 (sparse), Y -> Y (sparse), in that insertion order.
    ``order="after"`` adds Y before X.  Returns (net, inputs of every window)."""
    N, T = ns_.nodes, ns_.topology
    from bindsnet_b200.network.monitors import Monitor

    net = ns_.Network(dt=1.0, batch_size=c.B, learning=True)
    X, Y = N.Input(c.ns, traces=True), _target(N, c.kind, c.nt)
    for name, l in ((("Y", Y), ("X", X)) if c.order == "after" else (("X", X), ("Y", Y))):
        net.add_layer(l, name)
    kw = dict(update_rule=ns_.learning.NoOp, weight_decay=c.wd) if c.wd >= 0 else {}
    net.add_connection(T.SparseConnection(X, Y, w=d["w"].clone(), b=None if d["b"] is None else d["b"].clone(), **kw), "X", "Y")
    inputs = {"X": d["x"]}
    if c.dense:
        Z = N.Input(20)
        net.add_layer(Z, "Z")
        net.add_connection(T.Connection(Z, Y, w=d["wz"].clone()), "Z", "Y")
        inputs["Z"] = d["z"]
    if c.two:
        Y2 = _target(N, "iff", c.two)
        net.add_layer(Y2, "Y2")
        net.add_connection(T.SparseConnection(X, Y2, w=d["w2"].clone(), **kw), "X", "Y2")
        net.add_monitor(Monitor(Y2, ["s", "v"], time=c.T), "Y2m")
    if c.rec:
        net.add_connection(T.SparseConnection(Y, Y, w=d["wr"].clone(), **kw), "Y", "Y")
    net.add_monitor(Monitor(Y, ["s", "v"], time=c.T), "Ym")
    return net, inputs


def snapshot(net) -> dict:
    out = {}
    for lname, layer in net.layers.items():
        Bz = layer.s.shape[0]
        out[f"L/{lname}/s"] = layer.s.reshape(Bz, -1).to(torch.uint8).cpu()
        for var in ("v", "refrac_count", "x", "i"):
            val = getattr(layer, var, None)
            if isinstance(val, torch.Tensor) and val.numel() > 0:
                out[f"L/{lname}/{var}"] = val.detach().reshape(Bz, -1).float().cpu().clone()
    for (s, t), cn in net.connections.items():
        w = cn.w.detach()
        if w.is_sparse:
            w = w.coalesce()
            out[f"C/{s}{t}/idx"] = w.indices().cpu().clone()
            out[f"C/{s}{t}/val"] = w.values().cpu().clone()
        else:
            out[f"C/{s}{t}/w"] = w.cpu().clone()
    for mname, m in net.monitors.items():
        for var in m.state_vars:
            out[f"M/{mname}/{var}"] = m.get(var).float().cpu().clone()
    return out


def run(ns_, c: SparseCase, d: dict, device: str = "cpu"):
    """``windows`` windows of T steps; returns (per-window snapshots, net)."""
    net, inputs = build(ns_, c, d)
    net.force_tier = 1
    if device != "cpu":
        net.to(device)
    outs = []
    for k in range(c.windows):
        x = {n: v[k * c.T:(k + 1) * c.T].to(device) for n, v in inputs.items()}
        net.run(inputs=x, time=c.T, one_step=c.one_step)
        outs.append(snapshot(net))
    return outs, net


# ---- which spikes each connection reads -----------------------------------------------------------------------------

@dataclass
class Conn:
    src: str
    tgt: str
    idx: torch.Tensor         # [2, nnz] stored positions (a dense connection: every position)
    val: torch.Tensor         # [nnz] float64 values
    shape: tuple
    b: object                 # bias or None
    sparse: bool

    def product(self, s: torch.Tensor, val: torch.Tensor = None) -> torch.Tensor:
        """Per sample of s [B, ns] (0 / 1, float64), the sum of ``val`` (default: the values) over the stored positions
        of the spiking sources.  A silent source contributes no term: an infinite value of one does not make the sum NaN
        as the 0 * inf of a dense product would."""
        val = self.val if val is None else val
        fin = torch.isfinite(val)
        m = torch.sparse_coo_tensor(self.idx.flip(0)[:, fin], val[fin], self.shape[::-1]).coalesce()
        out = torch.sparse.mm(m, s.T).T
        for p in (~fin).nonzero().flatten().tolist():
            i, j = int(self.idx[0, p]), int(self.idx[1, p])
            out[:, j] = out[:, j] + torch.where(s[:, i] > 0, val[p], torch.zeros((), dtype=val.dtype))
        return out


def _conns(c: SparseCase, d: dict) -> list:
    """Every connection in insertion order."""
    def sp(src, tgt, w, b):
        w = w.coalesce()
        return Conn(src, tgt, w.indices(), w.values().to(torch.float64), tuple(w.shape), b, True)
    out = [sp("X", "Y", d["w"], d["b"])]
    if c.dense:
        wz = d["wz"]
        out.append(Conn("Z", "Y", torch.ones(wz.shape).nonzero().T, wz.reshape(-1).to(torch.float64), tuple(wz.shape), None, False))
    if c.two:
        out.append(sp("X", "Y2", d["w2"], None))
    if c.rec:
        out.append(sp("Y", "Y", d["wr"], None))
    return out


def _layer_order(c: SparseCase) -> list:
    names = ["Y", "X"] if c.order == "after" else ["X", "Y"]
    return names + (["Z"] if c.dense else []) + (["Y2"] if c.two else [])


def reads_current(c: SparseCase, src: str, tgt: str) -> bool:
    """One-step mode: a connection reads its source's spikes of this step when the source comes first in the layers'
    insertion order (network.py:383-396; phase_sparse's ``cur``)."""
    order = _layer_order(c)
    return c.one_step and order.index(src) < order.index(tgt)


def read_spikes(c: SparseCase, d: dict, src: str, tgt: str, rasters: dict) -> torch.Tensor:
    """[steps, B, ns] bool: the source spikes the connection reads at each step (s(-1) of the first window is zero)."""
    steps = c.T * c.windows
    s = {"X": d["x"], "Z": d.get("z")}.get(src)
    s = (s if s is not None else rasters[src]).bool()
    if reads_current(c, src, tgt):
        return s
    return torch.cat([torch.zeros(1, *s.shape[1:], dtype=torch.bool), s[:steps - 1]])


# ---- path table ---------------------------------------------------------------------------------------------------

def paths(c: SparseCase, d: dict, rasters: dict = None) -> dict:
    """Which side of each switch of sparse_block_width / plan_units / sparse_prepass / phase_sparse the case takes.
    ``rasters``: the non-input layers' spikes (a recurrent source); without them a recurrent connection is left out."""
    out = dict(counts=set(), entries=set(), late_row=False, col0=False, col_edge=False, col_edge_wide=False, col_last=False,
               empty_row=False, empty_col=False, anyf_skip=False, step0_slot2=False, cur=False, prev_one_step=False,
               all_group=False)
    widths = []
    for k in _conns(c, d):
        if not k.sparse:
            continue
        (ns, nt), nnz = k.shape, k.idx.shape[1]
        bw, stop = block_width(ns, nt, c.B, nnz)
        nb = _ceil(nt, bw)
        widths.append(bw)
        if (k.src, k.tgt) == ("X", "Y"):
            out.update(bw=bw, stop=stop, nb=nb, partial=nt % bw != 0, nnz0=nnz == 0, words_gt32=_ceil(ns, 32) > 32, nb_gt1=nb > 1)
        cur = reads_current(c, k.src, k.tgt)
        out["cur"] |= cur
        out["prev_one_step"] |= c.one_step and not cur
        anyf = _ceil(ns, 32) > 32
        out["step0_slot2"] |= anyf and not cur
        if k.src == "Y" and rasters is None:
            continue
        s = read_spikes(c, d, k.src, k.tgt, rasters or {})
        steps, B = s.shape[:2]
        ii, jj = k.idx
        out["empty_row"] |= bool((torch.bincount(ii, minlength=ns) == 0).any())
        out["empty_col"] |= bool((torch.bincount(jj, minlength=nt) == 0).any())
        blk = torch.zeros(ns, nb, dtype=torch.int64)   # entries of each row in each block
        blk.index_put_((ii, jj // bw), torch.ones_like(ii), accumulate=True)
        edge = torch.zeros(nt, dtype=torch.bool)
        edge[bw - 1::bw] = True
        for t in range(steps):
            for b in range(B):
                on = s[t, b]
                if anyf and not bool(on.any()) and (cur or t > 0):
                    out["anyf_skip"] = True
                for g0 in range(0, ns, GROUP):
                    n = int(on[g0:g0 + GROUP].sum())
                    out["counts"].add(n)
                    out["all_group"] |= n == min(GROUP, ns - g0) and n > 1
                rows = on.nonzero().flatten()
                if rows.numel() == 0:
                    continue
                rb = blk[rows]
                out["entries"].update(int(v) for v in rb.flatten().unique())
                out["late_row"] |= nb > 1 and bool(((rb[:, 0] == 0) & (rb.sum(1) > 0)).any())
                cols = jj[on[ii]]
                if cols.numel():
                    out["col0"] |= bool((cols == 0).any())
                    out["col_last"] |= bool((cols == nt - 1).any())
                    hit = bool(edge[cols].any())
                    out["col_edge"] |= hit
                    out["col_edge_wide"] |= hit and bw > 128
    out["two_widths"] = len(set(widths)) > 1
    out["b_tail"] = c.B % GEN_WARPS
    out["windows"] = c.windows
    return out


def check_claims(c, p: dict):
    for k, side in c.claims:
        assert p[k] == side, f"{c.name}: claims {k} = {side}, the mirror says {p[k]}"


# ---- float64 restatement --------------------------------------------------------------------------------------------

def lif_step_err(dec, E, a, rest, I, Vn):
    """tests/param_edges.py's bound of one LIF step (its module docstring, applied in ``ref_pn``): ``a`` = decay
    (v - rest), ``I`` the exact input, ``Vn`` the new voltage, ``E`` the bound v carried in."""
    return dec * (1 + DECAY_REL) * E + gamma(5) * (a.abs() + rest.abs() + I.abs() + Vn.abs()) + DECAY_REL * a.abs()


def _exp64(tc: float) -> float:
    return float(torch.exp(-1.0 / torch.tensor(tc, dtype=torch.float32).to(torch.float64)))


def decay_factor(wd: float) -> float:
    """learning.py:85-94: w *= 1 - wd when that is non-zero, as the fp32 factor the kernel holds; 1.0 (no rule, wd = 0,
    wd = 1): nothing changes."""
    if wd < 0 or wd == 0.0 or wd == 1.0:
        return 1.0
    return f32(1.0 - wd)


def ref_values(wd: float, w: torch.Tensor, steps: int):
    """A sparse connection's stored values after ``steps`` decays, float64, and their bound (an exact factor of +-1
    leaves them exact)."""
    f = decay_factor(wd)
    v = w.coalesce().values().to(torch.float64) * f ** steps
    return v, (torch.zeros_like(v) if f in (1.0, -1.0) else gamma(steps) * v.abs())


def ref_window(c: SparseCase, d: dict, outs: list) -> dict:
    """Every target teacher-forced with the oracle's spikes (``outs``: per-window snapshots, whose monitors hold s and v
    of every step).  Returns per target {"v": [steps, B, n], "v_err", "i", "i_err", "rc", "margin_ok", "raster_ok",
    "min_margin"}."""
    f64 = torch.float64
    steps, B = c.T * c.windows, c.B
    rasters = {"Y": torch.cat([o["M/Ym/s"] for o in outs]).reshape(steps, B, c.nt).bool()}
    kinds = {"Y": c.kind}
    if c.two:
        rasters["Y2"] = torch.cat([o["M/Y2m/s"] for o in outs]).reshape(steps, B, c.two).bool()
        kinds["Y2"] = "iff"
    conns = _conns(c, d)
    fac = decay_factor(c.wd)
    exact_decay = fac in (1.0, -1.0)
    dec, idec, rest = _exp64(20.0), _exp64(2.0), -65.0
    res = {}
    for tgt, kind in kinds.items():
        n = rasters[tgt].shape[2]
        ins = [(k, read_spikes(c, d, k.src, k.tgt, rasters).to(f64)) for k in conns if k.tgt == tgt]
        V = torch.full((B, n), -64.0 if kind == "iff" else rest, dtype=f64)   # (IFNodes start at reset, nodes.py:403-410)
        E, RC = torch.zeros(B, n, dtype=f64), torch.zeros(B, n, dtype=f64)
        I, EI = torch.zeros(B, n, dtype=f64), torch.zeros(B, n, dtype=f64)
        REST = torch.full((B, n), rest, dtype=f64)
        thr = THRESH[kind]
        r = dict(v=[], v_err=[], margin_ok=True, raster_ok=True, min_margin=np.inf)
        for t in range(steps):
            x, ab, cnt = (torch.zeros(B, n, dtype=f64) for _ in range(3))
            for k, s in ins:
                val = k.val * fac ** t if k.sparse else k.val
                x = x + k.product(s[t], val)
                ab = ab + k.product(s[t], val.abs())
                cnt = cnt + k.product(s[t], torch.ones_like(val))
                if k.b is not None:
                    x = x + k.b.to(f64)
                    ab = ab + k.b.to(f64).abs()
                    cnt = cnt + 1
            ex = gamma(cnt + 2 + (0 if exact_decay else t)) * ab
            if kind == "iff":
                gate = (RC <= 0).to(f64)
                Vn = V + gate * x
                E = E + U32 * Vn.abs() + gate * ex
                RC = RC - 1.0
            elif kind == "lif":
                gate = (RC <= 0).to(f64)
                a = dec * (V - rest)
                Vn = a + rest + gate * x
                E = lif_step_err(dec, E, a, REST, gate * x, Vn) + gate * ex
                RC = RC - 1.0
            else:
                Ip = idec * I
                I = Ip + x
                EI = idec * (1 + gamma(5)) * EI + gamma(5) * (Ip.abs() + I.abs()) + ex
                RC = RC - 1.0
                gate = (RC <= 0).to(f64)
                a = dec * (V - rest)
                Vn = a + rest + gate * I
                E = lif_step_err(dec, E, a, REST, gate * I, Vn) + gate * EI
            fin = torch.isfinite(Vn) & torch.isfinite(E)
            gap = (Vn - thr).abs() - E
            if bool(fin.any()):
                r["min_margin"] = min(r["min_margin"], float(gap[fin].min()))
                r["margin_ok"] &= not bool((gap[fin] <= 0).any())
            spk = Vn >= thr
            r["raster_ok"] &= torch.equal(spk, rasters[tgt][t])
            RC = torch.where(spk, torch.full((), 2.0, dtype=f64), RC)
            V = torch.where(spk, torch.full((), -64.0, dtype=f64), Vn)
            E = torch.where(spk, torch.zeros((), dtype=f64), E)
            r["v"].append(V.clone())
            r["v_err"].append(E.clone())
        r.update(v=torch.stack(r["v"]), v_err=torch.stack(r["v_err"]), rc=RC, i=I, i_err=EI)
        res[tgt] = r
    return res


# ---- the single operators --------------------------------------------------------------------------------------------

@dataclass(frozen=True)
class OpCase:
    ns: int
    nt: int
    B: int
    density: float = 0.1
    wd: float = 0.1
    values: str = "mixed"
    claims: tuple = ()

    @property
    def name(self) -> str:
        return f"op_{self.ns}x{self.nt}_b{self.B}_d{self.density:g}_wd{self.wd:g}" + (f"_{self.values}" if self.values != "mixed" else "")


OP_CASES = [
    OpCase(40, 33, 1, claims=(("nt_tail", True), ("grid_y_wraps", False))),
    OpCase(300, 100, 8, wd=2.0, values="zeros", claims=(("nt_tail", True),)),
    OpCase(70, 64, 513, wd=1.0, claims=(("grid_y_wraps", True), ("nt_tail", False))),
    OpCase(60, 45, 16, values="inf", wd=0.0),
    OpCase(1300, 1000, 2, density=1.0, wd=0.1, claims=(("update_blocks_capped", True),)),
]


def draw_op(c: OpCase) -> dict:
    g = torch.Generator().manual_seed(911 + c.ns + 7 * c.nt + 13 * c.B)
    mask = torch.rand(c.ns, c.nt, generator=g) < c.density
    w = _values(mask.nonzero().T, (c.ns, c.nt), c.values, g, 2.0)
    s = torch.rand(c.B, c.ns, generator=g) < 0.3
    s[0] = False   # a silent sample
    return dict(w=w, b=torch.rand(c.nt, generator=g) - 0.5, s=s)


def op_paths(c: OpCase, d: dict) -> dict:
    nnz = d["w"]._nnz()
    return dict(nt_tail=c.nt % 32 != 0, grid_y_wraps=_ceil(c.B, GEN_WARPS) > OP_GRID_Y,
                update_blocks_capped=_ceil(nnz, 1024) > OP_UPDATE_BLOCKS)


def run_op(ns_, c: OpCase, d: dict, device: str = "cpu"):
    """connection.compute(s), then connection.update() (NoOp decay).  Returns {"out", "val"}."""
    N = ns_.nodes
    X, Y = N.Input(c.ns), N.IFNodes(c.nt)
    conn = ns_.topology.SparseConnection(X, Y, w=d["w"].clone(), b=d["b"].clone(), update_rule=ns_.learning.NoOp,
                                         weight_decay=c.wd)
    for l in (X, Y):
        l.compute_decays(1.0)
        l.set_batch_size(c.B)
    if device != "cpu":
        for m in (X, Y, conn):
            m.to(device)
    out = conn.compute(d["s"].to(device)).cpu().clone()
    X.s = d["s"].to(device).clone()
    conn.update(learning=True)
    return dict(out=out, val=conn.w.detach().coalesce().values().cpu().clone())


def ref_op(c: OpCase, d: dict):
    """(out, bound, stored values after one decay, bound)."""
    w = d["w"].coalesce()
    k = Conn("X", "Y", w.indices(), w.values().to(torch.float64), tuple(w.shape), d["b"], True)
    s = d["s"].to(torch.float64)
    b = d["b"].to(torch.float64)
    out = k.product(s) + b
    cnt = k.product(s, torch.ones_like(k.val)) + 1
    bound = gamma(cnt) * (k.product(s, k.val.abs()) + b.abs())
    v = k.val * decay_factor(c.wd)
    return out, bound, v, U32 * v.abs()
