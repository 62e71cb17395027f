"""Heterogeneous graphs — GNNHeteroGraph (GNNGraphs/src/gnnheterograph/gnnheterograph.jl:85-155) with its queries,
transforms and generators (gnnheterograph/query.jl, transform.jl, generate.jl), and HeteroGraphConv
(GraphNeuralNetworks/src/layers/heteroconv.jl:40-86).

Node types are strings and edge types ``(src_t, rel, dst_t)`` tuples of strings (the reference uses symbols).  Each
relation is a COO ``(s, t[, w])`` with 1-based ids and owns one lazily built device plan with ``num_src =
num_nodes[src_t]`` and ``num_dst = num_nodes[dst_t]``: the bipartite plans of the engine.  ``edge_type_subgraph``
shares the parent's relations, plans included, so a layer applied relation by relation builds each plan once.

A one-relation heterograph goes through the message-passing framework and the relation-wise layers like a GNNGraph:
results have num_dst rows and pullbacks num_src rows (``graph.num_src_dst``).
"""
from __future__ import annotations

import operator
from typing import Optional

import numpy as np
import torch

from . import _lib
from . import graph as _graph
from .graph import GNNGraph, _as_index, _Plan, _make_plan, _stream, colmajor


def _is_etype(k) -> bool:
    return isinstance(k, tuple) and len(k) == 3 and all(isinstance(v, str) for v in k)


def _is_pair(p) -> bool:
    return isinstance(p, tuple) and len(p) == 2 and _is_etype(p[0])


class _Relation:
    """One edge type's COO and its device plan (built once, on first use)."""

    def __init__(self, s, t, w, num_src: int, num_dst: int):
        self.s, self.t = s, t
        self.w = None if w is None else torch.as_tensor(w, dtype=torch.float32).to(s.device).contiguous()
        self.num_edges = int(s.numel())
        assert self.w is None or self.w.numel() == self.num_edges, "edge weight length must equal num_edges"
        self.num_src, self.num_dst = int(num_src), int(num_dst)
        self._plan: Optional[_Plan] = None
        self._loops: Optional["_Relation"] = None

    def plan(self, device=None) -> _Plan:
        """Build (once) and return the relation's plan.  Raises AssertionError on out-of-range indices."""
        if self._plan is None:
            self._plan = _make_plan(self.s, self.t, self.num_edges, self.num_src, self.num_dst, device)
        return self._plan


def _features(d, default: str):
    if d is None:
        return {}
    if isinstance(d, torch.Tensor) or isinstance(d, np.ndarray):
        return {default: d}
    if isinstance(d, tuple) and hasattr(d, "_fields"):
        return dict(d._asdict())
    if isinstance(d, dict):
        return dict(d)
    return {default: d}


def _typed(d, key_ok) -> dict:
    """a dict, an iterable of pairs or a single pair keyed by types"""
    if d is None:
        return {}
    if isinstance(d, dict):
        return dict(d)
    if isinstance(d, tuple) and len(d) == 2 and key_ok(d[0]):
        return {d[0]: d[1]}
    return dict(d)


class GNNHeteroGraph:
    """COO heterograph (gnnheterograph.jl:85-155).

    ``GNNHeteroGraph()`` (empty), ``GNNHeteroGraph({et: (s, t[, w]), ...})``, ``GNNHeteroGraph((et, (s, t)), ...)``
    and ``GNNHeteroGraph([(et, (s, t)), ...])``; ``num_nodes`` as a dict or pairs, inferred per type from the largest
    index otherwise.  ``g["A"]`` is node type A's ndata, ``g[("A", "r", "B")]`` the relation's edata."""

    is_hetero = True

    def __init__(self, *data, num_nodes=None, graph_indicator=None, ndata=None, edata=None, gdata=None,
                 num_graphs: Optional[int] = None, device=None):
        if len(data) == 1 and isinstance(data[0], dict):
            items = list(data[0].items())
        elif len(data) == 1 and not _is_pair(data[0]) and isinstance(data[0], (list, tuple)):
            items = list(data[0])
        else:
            items = list(data)
        for k, _ in items:
            if not _is_etype(k):
                raise ValueError("Keys of data must be tuples of the form (source_type, edge_type, target_type)")
        given = {k: int(v) for k, v in _typed(num_nodes, lambda k: isinstance(k, str)).items()}
        coo = {}
        for et, st in items:
            st = tuple(st)
            s, t = _as_index(st[0], device).reshape(-1), _as_index(st[1], device).reshape(-1)
            assert s.numel() == t.numel(), "s and t must be vectors of equal length"
            coo[et] = (s, t, st[2] if len(st) > 2 else None)
        self.etypes = list(coo)
        self.ntypes = []
        for (a, _, b) in self.etypes:
            for nt in (a, b):
                if nt not in self.ntypes:
                    self.ntypes.append(nt)
        for nt in given:
            if nt not in self.ntypes:
                self.ntypes.append(nt)
        self.num_nodes = {}
        for nt in self.ntypes:
            if nt in given:
                self.num_nodes[nt] = given[nt]
                continue
            m = 0
            for (a, _, b), (s, t, _) in coo.items():
                if a == nt and s.numel():
                    m = max(m, int(s.max()))
                if b == nt and t.numel():
                    m = max(m, int(t.max()))
            self.num_nodes[nt] = m
        self._rels = {et: _Relation(s, t, w, self.num_nodes[et[0]], self.num_nodes[et[2]])
                      for et, (s, t, w) in coo.items()}
        self.graph_indicator = None if graph_indicator is None else dict(graph_indicator)
        if num_graphs is None:
            num_graphs = (max(int(torch.as_tensor(v).max()) for v in self.graph_indicator.values())
                          if self.graph_indicator else 1)
        self.num_graphs = int(num_graphs)
        nd, ed = _typed(ndata, lambda k: isinstance(k, str)), _typed(edata, _is_etype)
        self.ndata = {nt: _features(nd.get(nt), "x") for nt in self.ntypes}
        self.edata = {et: _features(ed.get(et), "e") for et in self.etypes}
        self.gdata = _features(gdata, "u")
        for nt, d in self.ndata.items():
            for k, v in d.items():
                assert v.shape[-1] == self.num_nodes[nt], f"ndata[{nt!r}].{k}: last dimension must be num_nodes"
        for et, d in self.edata.items():
            for k, v in d.items():
                assert v.shape[-1] == self.num_edges[et], f"edata[{et!r}].{k}: last dimension must be num_edges"

    # -- construction from parts (shares relations and their plans)
    @classmethod
    def _from(cls, rels: dict, num_nodes: dict, ntypes, *, graph_indicator=None, ndata=None, edata=None, gdata=None,
              num_graphs: int = 1) -> "GNNHeteroGraph":
        g = cls.__new__(cls)
        g._rels = dict(rels)
        g.etypes = list(rels)
        g.ntypes = list(ntypes)
        g.num_nodes = dict(num_nodes)
        g.graph_indicator = graph_indicator
        g.num_graphs = int(num_graphs)
        g.ndata = {nt: dict((ndata or {}).get(nt, {})) for nt in g.ntypes}
        g.edata = {et: dict((edata or {}).get(et, {})) for et in g.etypes}
        g.gdata = dict(gdata or {})
        return g

    @property
    def num_edges(self) -> dict:
        return {et: r.num_edges for et, r in self._rels.items()}

    @property
    def device(self):
        for r in self._rels.values():
            return r.s.device
        return torch.device("cpu")

    def relation(self, et) -> _Relation:
        assert et in self._rels, f"Edge type {et} not found in graph"
        return self._rels[et]

    def only_relation(self) -> _Relation:
        assert len(self.etypes) == 1, \
            f"message passing needs a heterograph of one edge type (got {len(self.etypes)}): use edge_type_subgraph"
        return self._rels[self.etypes[0]]

    def plan(self, et=None) -> _Plan:
        return (self.only_relation() if et is None else self.relation(et)).plan()

    def __getitem__(self, key):
        if isinstance(key, str):
            return self.ndata.setdefault(key, {})
        return self.edata.setdefault(key, {})

    def __repr__(self):
        return f"GNNHeteroGraph(num_nodes={self.num_nodes}, num_edges={self.num_edges})"


# ------------------------------------------------------------------------------------------------- queries
def num_edge_types(g) -> int:
    """gnnheterograph.jl:230-242: 1 for a GNNGraph."""
    return len(g.etypes) if _graph._is_hetero(g) else 1


def num_node_types(g) -> int:
    return len(g.ntypes) if _graph._is_hetero(g) else 1


def edge_type_subgraph(g: GNNHeteroGraph, edge_ts) -> GNNHeteroGraph:
    """gnnheterograph.jl:250-271: the relations of `edge_ts` (one type or a list), sharing g's relations and plans."""
    ets = [edge_ts] if _is_etype(edge_ts) else list(edge_ts)
    for et in ets:
        assert et in g._rels, f"Edge type {et} not found in graph"
    nts = []
    for a, _, b in ets:
        for nt in (a, b):
            if nt not in nts:
                nts.append(nt)
    gi = None if g.graph_indicator is None else {nt: g.graph_indicator[nt] for nt in nts if nt in g.graph_indicator}
    return GNNHeteroGraph._from({et: g._rels[et] for et in ets}, {nt: g.num_nodes[nt] for nt in nts}, nts,
                                graph_indicator=gi, ndata={nt: g.ndata[nt] for nt in nts if nt in g.ndata},
                                edata={et: g.edata[et] for et in ets if et in g.edata}, gdata=g.gdata,
                                num_graphs=g.num_graphs)


def edge_index(g: GNNHeteroGraph, et=None):
    """gnnheterograph/query.jl:9-10: (s, t) of `et` (of the only relation without it)."""
    r = g.only_relation() if et is None else g.relation(et)
    return r.s, r.t


def get_edge_weight(g: GNNHeteroGraph, et=None):
    r = g.only_relation() if et is None else g.relation(et)
    return r.w


def has_edge(g, *args) -> bool:
    """has_edge(g, edge_t, i, j) (gnnheterograph/query.jl:34-37); has_edge(g, i, j) for a GNNGraph."""
    if _graph._is_hetero(g):
        et, i, j = args
        s, t = edge_index(g, et)
    else:
        i, j = args
        s, t = g.s, g.t
    return bool(((s == int(i)) & (t == int(j))).any())


def degree(g: GNNHeteroGraph, et, T=None, *, dir: str = "out") -> torch.Tensor:
    """gnnheterograph/query.jl:55-68: unweighted degrees of relation `et`, over its source type (dir="out") or its
    target type (dir="in").  The node type comes from `et` (the reference takes g.ntypes[1 or 2])."""
    assert dir in ("in", "out"), 'a relation has dir "in" or "out"'
    r = g.relation(et)
    p = r.plan()
    n = r.num_dst if dir == "in" else r.num_src
    out = torch.empty(n, dtype=torch.float32, device=p.device)
    with torch.cuda.device(p.device):
        _lib.check(_lib.lib.gnnb_degree(p.h, _lib.DIR_IN if dir == "in" else _lib.DIR_OUT, None, out.data_ptr(),
                                   _stream(p.device)))
    return out.to(r.s.dtype if T is None else T)


def graph_indicator(g: GNNHeteroGraph, node_t=None):
    """gnnheterograph/query.jl:81-98: the dict of indicators (None for one graph), or node type `node_t`'s."""
    if node_t is None:
        return g.graph_indicator
    assert node_t in g.ntypes
    if g.graph_indicator is None:
        return torch.ones(g.num_nodes[node_t], dtype=torch.int64, device=g.device)
    return g.graph_indicator[node_t]


# ------------------------------------------------------------------------------------------------- transforms
def _loops(r: _Relation, n: int) -> _Relation:
    """r plus one loop per node (weights padded with 1), cached on r; the plan is derived from r's on the device"""
    if r._loops is not None:
        return r._loops
    nodes = torch.arange(1, n + 1, dtype=r.s.dtype, device=r.s.device)
    w = None if r.w is None else torch.cat([r.w, torch.ones(n, dtype=r.w.dtype, device=r.w.device)])
    h = _Relation(torch.cat([r.s, nodes]), torch.cat([r.t, nodes]), w, n, n)
    if _lib.device_count() > 0:
        import ctypes as C
        p = r.plan()
        hh = C.c_void_p()
        with torch.cuda.device(p.device):
            _lib.check(_lib.lib.gnnb_graph_add_self_loops(p.h, C.byref(hh), _stream(p.device)))
        h._plan = _Plan(hh.value, p.device)
    r._loops = h
    return h


def add_self_loops(g: GNNHeteroGraph, et=None) -> GNNHeteroGraph:
    """gnnheterograph/transform.jl:20-76: a loop per node on `et` when its source and target types are one (g itself
    otherwise); without `et`, on every such relation."""
    if et is None:
        for e in list(g.etypes):
            g = add_self_loops(g, e)
        return g
    a, _, b = et
    if a != b:
        return g
    n = g.num_nodes.get(a, 0)
    rels = dict(g._rels)
    if et in rels:
        rels[et] = _loops(rels[et], n)
    else:
        nodes = torch.arange(1, n + 1, dtype=torch.int64, device=g.device)
        rels[et] = _Relation(nodes, nodes.clone(), None, n, n)
    ntypes = g.ntypes + ([a] if a not in g.ntypes else [])
    return GNNHeteroGraph._from(rels, {**g.num_nodes, a: n}, ntypes, graph_indicator=g.graph_indicator,
                                ndata=g.ndata, edata=g.edata, gdata=g.gdata, num_graphs=g.num_graphs)


def add_edges(g, *args, edata=None, num_nodes=None, **kws):
    """add_edges(g, et, s, t), add_edges(g, (et, (s, t[, w]))) with edata= and num_nodes=
    (gnnheterograph/transform.jl:92-163); a GNNGraph goes to the homogeneous add_edges."""
    if not _graph._is_hetero(g):
        if num_nodes is not None:
            raise TypeError("add_edges(g::GNNGraph, ...) takes no num_nodes (the node count follows the new ids)")
        from .linkpred import add_edges as homog
        return homog(g, *args, edata=edata, **kws)
    if kws:
        raise TypeError(f"add_edges(g::GNNHeteroGraph, ...) got unexpected keyword arguments {sorted(kws)}")
    if len(args) == 1:
        et, data = args[0]
    else:
        et, data = args[0], tuple(args[1:])
    data = tuple(data)
    dev = g.device
    snew, tnew = _as_index(data[0], dev).reshape(-1), _as_index(data[1], dev).reshape(-1)
    wnew = data[2] if len(data) > 2 else None
    assert snew.numel() == tnew.numel(), "s and t must have the same length"
    if snew.numel() == 0:
        return g
    assert int(snew.min()) >= 1 and int(tnew.min()) >= 1, "node ids are 1-based"
    nn = _typed(num_nodes, lambda k: isinstance(k, str))
    counts, ntypes = dict(g.num_nodes), list(g.ntypes)
    rels, ed = dict(g._rels), {k: dict(v) for k, v in g.edata.items()}
    new_ed = _features(edata, "e")
    if et not in rels:
        for nt, ids in ((et[0], snew), (et[2], tnew)):
            if nt not in ntypes:
                ntypes.append(nt)
                counts[nt] = int(nn[nt]) if nt in nn else int(ids.max())
        s, t, w = snew, tnew, wnew
        ed[et] = new_ed
    else:
        r = rels[et]
        s, t = torch.cat([r.s, snew.to(r.s.dtype)]), torch.cat([r.t, tnew.to(r.t.dtype)])
        w = None
        if r.w is not None or wnew is not None:
            w_old = r.w if r.w is not None else torch.ones(r.num_edges, dtype=torch.float32, device=dev)
            w_new = (torch.as_tensor(wnew, dtype=torch.float32).to(dev) if wnew is not None
                     else torch.ones(snew.numel(), dtype=torch.float32, device=dev))
            w = torch.cat([w_old, w_new])
        old = ed.get(et, {})
        ed[et] = {k: torch.cat([colmajor(v), torch.as_tensor(new_ed[k]).to(v.device, v.dtype)], dim=-1)
                  for k, v in old.items() if k in new_ed}
    counts[et[0]] = max(counts[et[0]], int(s.max()))
    counts[et[2]] = max(counts[et[2]], int(t.max()))
    rels[et] = _Relation(s, t, w, counts[et[0]], counts[et[2]])
    for e, r in list(rels.items()):              # relations whose node counts grew get a plan of the new size
        if e != et and (r.num_src != counts[e[0]] or r.num_dst != counts[e[2]]):
            rels[e] = _Relation(r.s, r.t, r.w, counts[e[0]], counts[e[2]])
    return GNNHeteroGraph._from(rels, counts, ntypes, graph_indicator=g.graph_indicator, ndata=g.ndata, edata=ed,
                                gdata=g.gdata, num_graphs=g.num_graphs)


def batch(graphs) -> GNNHeteroGraph:
    """gnnheterograph/transform.jl:165-230: per-type node offsets, relations concatenated in graph order, a
    graph_indicator for every node type.  Every graph must hold one graph (as the reference asserts)."""
    gs = list(graphs)
    assert len(gs) > 0
    assert all(g.num_graphs == 1 for g in gs), "batch of heterographs needs num_graphs == 1 for each"
    ntypes, etypes = [], []
    for g in gs:
        ntypes += [nt for nt in g.ntypes if nt not in ntypes]
        etypes += [et for et in g.etypes if et not in etypes]
    dev = gs[0].device
    off = {nt: np.cumsum([0] + [g.num_nodes.get(nt, 0) for g in gs]) for nt in ntypes}
    counts = {nt: int(off[nt][-1]) for nt in ntypes}
    rels = {}
    for et in etypes:
        a, _, b = et
        parts = [(i, g._rels[et]) for i, g in enumerate(gs) if et in g._rels]
        s = torch.cat([r.s.to(torch.int64) + int(off[a][i]) for i, r in parts])
        t = torch.cat([r.t.to(torch.int64) + int(off[b][i]) for i, r in parts])
        ws = [r.w for _, r in parts]
        w = None if any(x is None for x in ws) else torch.cat(ws)
        rels[et] = _Relation(s, t, w, counts[a], counts[b])
    gi = {nt: torch.cat([torch.full((g.num_nodes.get(nt, 0),), i + 1, dtype=torch.int64, device=dev)
                         for i, g in enumerate(gs)]) for nt in ntypes}

    def cat(dicts):
        keys = [k for k in dicts[0] if all(k in d for d in dicts)]
        return {k: torch.cat([colmajor(d[k]) for d in dicts], dim=-1) for k in keys}

    nd = {nt: cat([g.ndata.get(nt, {}) for g in gs]) for nt in ntypes}
    ed = {et: cat([g.edata.get(et, {}) for g in gs if et in g._rels]) for et in etypes}
    return GNNHeteroGraph._from(rels, counts, ntypes, graph_indicator=gi, ndata=nd, edata=ed, num_graphs=len(gs))


# ------------------------------------------------------------------------------------------------- generators
def _rand_edges(n1: int, n2: int, m: int, seed, dev):
    """m distinct (s, t) of [1, n1] x [1, n2], without replacement (GNNGraphs/src/utils.jl:286-291), drawn on the
    device from the bipartite code space (the generator rand_graph uses)."""
    from .linkpred import _decode, sample_codes, space_size
    M = space_size(_lib.CODES_BIPARTITE, n1, n2)
    assert 0 <= m <= M, f"{m} distinct edges asked of {n1} x {n2} node pairs"
    return _decode(_lib.CODES_BIPARTITE, n1, n2, sample_codes(M, m, seed=seed, device=dev), dev)


def rand_heterograph(n, m, *, bidirected: bool = False, seed=None, device=None, **kws) -> GNNHeteroGraph:
    """gnnheterograph/generate.jl: `n` node counts and `m` edge counts per type (dicts or pairs); m[et] distinct random
    edges per relation.  bidirected: each relation (a, r, b) also gets (b, r, a) as its mirror (equal counts)."""
    n = _typed(n, lambda k: isinstance(k, str))
    m = _typed(m, _is_etype)
    dev = torch.device(device) if device is not None else _graph._compute_device(torch.empty(0))
    base = None if seed is None else int(seed)
    data = {}
    for i, (et, k) in enumerate(m.items()):
        rev = (et[2], et[1], et[0])
        if bidirected and rev in data:
            assert int(m[rev]) == int(k), "Number of edges must be the same in reverse edge types for bidirected graphs."
            continue
        s, t = _rand_edges(int(n[et[0]]), int(n[et[2]]), int(k), None if base is None else base + i, dev)
        data[et] = (s, t)
        if bidirected:
            if rev in m:
                assert int(m[rev]) == int(k), \
                    "Number of edges must be the same in reverse edge types for bidirected graphs."
            data[rev] = (t, s)
    return GNNHeteroGraph(data, num_nodes=n, **kws)


def rand_bipartite_heterograph(n, m, *, bidirected: bool = True, node_t=("A", "B"), edge_t: str = "to", seed=None,
                               **kws) -> GNNHeteroGraph:
    """gnnheterograph/generate.jl: node types node_t = (n1, n2) nodes, relations (A, to, B) and (B, to, A) with m
    (or (m12, m21)) edges."""
    n1, n2 = n
    m12, m21 = (m, m) if isinstance(m, int) else m
    return rand_heterograph({node_t[0]: n1, node_t[1]: n2},
                            {(node_t[0], edge_t, node_t[1]): m12, (node_t[1], edge_t, node_t[0]): m21},
                            bidirected=bidirected, seed=seed, **kws)


# ------------------------------------------------------------------------------------------------- HeteroGraphConv
class HeteroGraphConv(torch.nn.Module):
    """HeteroGraphConv(pairs...; aggr=+) — heteroconv.jl:40-86.  Built from (edge_t, layer) pairs, a list of them or a
    dict.  Each layer runs on edge_type_subgraph(g, edge_t) with (x[src_t], x[dst_t]); the outputs are folded per
    destination type with `aggr` (any binary function) in layer order.  Returns a dict keyed by destination type in
    first-appearance order; types no relation targets are absent."""

    def __init__(self, *itr, aggr=operator.add):
        super().__init__()
        if len(itr) == 1 and isinstance(itr[0], dict):
            pairs = list(itr[0].items())
        elif len(itr) == 1 and not _is_pair(itr[0]):
            pairs = list(itr[0])
        else:
            pairs = list(itr)
        assert all(_is_pair(p) for p in pairs), "HeteroGraphConv takes (edge_type, layer) pairs"
        self.etypes = [p[0] for p in pairs]
        self.layers = torch.nn.ModuleList([p[1] for p in pairs])
        self.aggr = aggr

    def forward(self, g: GNNHeteroGraph, x) -> dict:
        get = (lambda k: getattr(x, k)) if (isinstance(x, tuple) and hasattr(x, "_fields")) else (lambda k: x[k])
        out = {}
        for layer, et in zip(self.layers, self.etypes):
            y = layer(edge_type_subgraph(g, et), (get(et[0]), get(et[2])))
            out[et[2]] = y if et[2] not in out else self.aggr(out[et[2]], y)
        return out

    def __repr__(self):
        return f"HeteroGraphConv(aggr={getattr(self.aggr, '__name__', self.aggr)}, etypes={self.etypes})"
