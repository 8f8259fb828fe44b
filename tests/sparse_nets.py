"""Networks with SparseConnections shared by tests/test_sparse_connection.py (CPU: oracle, emulated kernel, live reference)
and tests/test_gpu_sparse.py (the CUDA library)."""
from __future__ import annotations

import torch

import helpers

T_LIVE, B_LIVE = 60, 3


def _pattern(n_src, n_tgt, density, scale, g, shift=0.0):
    """A dense [n_src, n_tgt] matrix that is zero outside a random pattern of the given density."""
    mask = torch.rand(n_src, n_tgt, generator=g) < density
    return ((torch.rand(n_src, n_tgt, generator=g) + shift) * scale) * mask


def live_net(ns, decay: bool, dense_recurrent: bool = False, dense_input: bool = False):
    """Input(64) -> SparseConnection (10 %, bias) -> LIFNodes(48), a second input Z -> LIF through a dense PostPre
    Connection, and a recurrent LIF -> LIF SparseConnection with negative weights, in that insertion order.
    ``decay``: both sparse connections carry learning.NoOp(weight_decay=0.1).  ``dense_*``: the same values as a dense
    Connection instead (the bit-identity check)."""
    g = torch.Generator().manual_seed(2024)
    w1 = _pattern(64, 48, 0.10, 9.0, g)
    w2 = _pattern(48, 48, 0.15, -4.0, g)
    wz = 0.3 * torch.rand(32, 48, generator=g)
    bias = 0.2 * torch.rand(48, generator=g)
    x = (torch.rand(T_LIVE, B_LIVE, 64, generator=g) < 0.12).to(torch.uint8)
    z = (torch.rand(T_LIVE, B_LIVE, 32, generator=g) < 0.1).to(torch.uint8)
    net = ns.Network(dt=1.0, batch_size=B_LIVE, learning=True)
    X, Z = ns.nodes.Input(64, traces=True), ns.nodes.Input(32, traces=True)
    Y = ns.nodes.LIFNodes(48, traces=True, thresh=-56.0, tc_decay=40.0, refrac=3)
    net.add_layer(X, "X"); net.add_layer(Z, "Z"); net.add_layer(Y, "Y")
    kw = dict(update_rule=ns.learning.NoOp, weight_decay=0.1) if decay else {}
    T = ns.topology
    net.add_connection(T.Connection(X, Y, w=w1, b=bias, **kw) if dense_input else T.SparseConnection(X, Y, w=w1.to_sparse(), b=bias, **kw),
                       "X", "Y")
    net.add_connection(T.Connection(Z, Y, w=wz, nu=(1e-3, 2e-3), update_rule=ns.learning.PostPre, wmin=0.0, wmax=1.0), "Z", "Y")
    net.add_connection(T.Connection(Y, Y, w=w2, **kw) if dense_recurrent else T.SparseConnection(Y, Y, w=w2.to_sparse(), **kw), "Y", "Y")
    mon = ns.monitors.Monitor(Y, ["s"], time=T_LIVE)
    net.add_monitor(mon, "Ys")
    return net, {"X": x, "Z": z}


def run_live(ns, decay: bool, **kw):
    net, inputs = live_net(ns, decay, **kw)
    net.run(inputs=inputs, time=T_LIVE)
    return net


def live_state(net) -> dict:
    out = {"Ys": net.monitors["Ys"].get("s").to(torch.uint8)}
    for l in ("X", "Y"):
        out[f"{l}/x"] = net.layers[l].x.clone()
    out["Y/v"] = net.layers["Y"].v.clone()
    out["Y/refrac_count"] = net.layers["Y"].refrac_count.clone()
    for (s, t), c in net.connections.items():
        w = c.w.detach()
        if w.is_sparse:
            w = w.coalesce()
            out[f"{s}{t}/idx"] = w.indices().clone()
            out[f"{s}{t}/val"] = w.values().clone()
        else:
            out[f"{s}{t}/w"] = w.clone()
    return out


def random_net(ns, seed: int):
    """A randomly drawn network around one or two SparseConnections: sizes that are not multiples of a column block,
    empty rows and columns, nnz = 0, a row with more entries than a block; IF / CurrentLIF / LIF targets, bias or none,
    NoOp decay or static.  Returns (net, inputs, spec)."""
    g = torch.Generator().manual_seed(1000 + seed)
    r = lambda k: int(torch.randint(0, k, (1,), generator=g))
    n_in, n_hid = [16, 70, 300][r(3)], [33, 130, 300][r(3)]
    B, T = [1, 3, 9][r(3)], [12, 25][r(2)]
    density = [0.0, 0.03, 0.2][r(3)] if seed % 4 else 0.0 if seed % 8 == 0 else 0.05
    kind = ["LIFNodes", "IFNodes", "CurrentLIFNodes"][r(3)]
    spec = dict(n_in=n_in, n_hid=n_hid, B=B, T=T, density=density, kind=kind, one_step=bool(r(2)), learning=bool(r(2)),
                decay=bool(r(2)), bias=bool(r(2)), recurrent=bool(r(2)))
    w1 = _pattern(n_in, n_hid, density, 6.0, g)
    if density > 0 and n_hid > 128:
        w1[r(n_in)] = 2.0 * torch.rand(n_hid, generator=g)           # a full row: more entries than a 128-column block
    w1[:, r(n_hid)] = 0.0                                             # an empty column
    w2 = _pattern(n_hid, n_hid, density, -3.0, g, shift=-0.2)
    x = (torch.rand(T, B, n_in, generator=g) < 0.25).to(torch.uint8)
    net = ns.Network(dt=1.0, batch_size=B, learning=spec["learning"])
    X = ns.nodes.Input(n_in, traces=True)
    Y = getattr(ns.nodes, kind)(n_hid, traces=True, thresh=-55.0 if kind != "IFNodes" else -54.0)
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    kw = dict(update_rule=ns.learning.NoOp, weight_decay=0.05) if spec["decay"] else {}
    b = torch.rand(n_hid, generator=g) if spec["bias"] else None
    net.add_connection(ns.topology.SparseConnection(X, Y, w=w1.to_sparse(), b=b, **kw), "X", "Y")
    if spec["recurrent"]:
        net.add_connection(ns.topology.SparseConnection(Y, Y, w=w2.to_sparse(), **kw), "Y", "Y")
    helpers.add_spike_monitors(net, T)
    return net, {"X": x}, spec


def big_index_net(ns):
    """n_src = n_tgt = 50 000 (n_src * n_tgt > 2**31) with about 10**4 stored entries, B = 2."""
    n, nnz, B = 50_000, 10_000, 2
    g = torch.Generator().manual_seed(5)
    flat = torch.unique(torch.randint(0, n * n, (nnz,), generator=g, dtype=torch.int64))
    flat[-1] = n * n - 1                                              # the last synapse of the matrix
    idx = torch.stack([flat // n, flat % n])
    w = torch.sparse_coo_tensor(idx, 30.0 * torch.rand(flat.numel(), generator=g), (n, n)).coalesce()
    x = (torch.rand(4, B, n, generator=g) < 0.3).to(torch.uint8)
    x[:, :, n - 1] = 1
    net = ns.Network(dt=1.0, batch_size=B, learning=True)
    X, Y = ns.nodes.Input(n), ns.nodes.LIFNodes(n)
    net.add_layer(X, "X"); net.add_layer(Y, "Y")
    net.add_connection(ns.topology.SparseConnection(X, Y, w=w, update_rule=ns.learning.NoOp, weight_decay=0.01), "X", "Y")
    helpers.add_spike_monitors(net, 4)
    return net, {"X": x}, 4


def sparse_values(net) -> dict:
    return {f"C/{s}->{t}/val": c.w.detach().coalesce().values().float().cpu().numpy()
            for (s, t), c in net.connections.items() if c.w.is_sparse}


def snapshot(net, T) -> dict:
    """helpers.snapshot with the stored values of the sparse connections instead of a dense w."""
    out = {}
    for lname, layer in net.layers.items():
        Bz = layer.s.shape[0]
        out[f"L/{lname}/s"] = layer.s.reshape(Bz, -1).to(torch.uint8).cpu().numpy()
        for var in ("v", "refrac_count", "x", "i"):
            val = getattr(layer, var, None)
            if isinstance(val, torch.Tensor) and val.numel() > 0:
                out[f"L/{lname}/{var}"] = val.detach().reshape(Bz, -1).float().cpu().numpy()
    for (s, t), c in net.connections.items():
        if not c.w.is_sparse:
            out[f"C/{s}->{t}/w"] = c.w.detach().float().cpu().numpy()
    out.update(sparse_values(net))
    if all(f"mon_{l}" in net.monitors for l in net.layers):
        out.update(helpers.spike_counts(net, T))
    return out


def reservoir(ns, n: int, p: float, B: int, T: int, seed: int = 0, dense: bool = False):
    """bench_sparse.py's reservoir, built on the CPU (``ns`` must be the b200 namespace)."""
    import bench_sparse

    assert ns.kind == "b200"
    return bench_sparse.build_reservoir(n, p, B, T, torch.device("cpu"), seed, dense)
