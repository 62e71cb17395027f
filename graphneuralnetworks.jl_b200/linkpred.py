"""Link prediction on the device: edge codes, random graphs, negative edges and edge splits.

    edge_encoding(s, t, n; directed, self_loops), edge_decoding(idx, n; ...)   GNNGraphs/src/utils.jl:189-268
    rand_graph(n, m; bidirected=true, edge_weight, seed)                      GNNGraphs/src/generate.jl:51-65
    negative_sample(g; num_neg_edges, bidirected, seed)                        GNNGraphs/src/transform.jl:890-929
    rand_edge_split(g, frac; bidirected, seed)                                 GNNGraphs/src/transform.jl:945-968
    perturb_edges(g, ratio; seed)                                              GNNGraphs/src/transform.jl:385-418
    add_edges(g, (s, t[, w]); edata)                                           GNNGraphs/src/transform.jl:319-353
    intersect(g1, g2)                                                          GNNGraphs/src/operators.jl:7-20
    dot_decoder(g, x), DotDecoder                                              GNNlib/src/layers/basic.jl:1-3

Every random choice here is one primitive, csrc/edgegen.cu's `gnnb_sample_codes`: the first m codes of a seeded
permutation π of a code space [0, M) that are not in a sorted exclusion set, in π order.  rand_graph takes m codes of
the space without self loops (undirected and mirrored when bidirected); negative_sample takes them from the same space
with the graph's own edges excluded; rand_edge_split permutes the edge ids; perturb_edges draws new directed edges.
The exclusion set is `gnnb_edge_codes_sorted` (encode, radix sort, one code per run), membership tests are
`gnnb_codes_member`.  Graphs given on the CPU are staged to the current CUDA device and the results live there.

Deliberate differences from the reference:
1. Order.  Sampled edges come in π order, not in ascending code order.
2. No truncation bias.  The reference's negative_sample draws about 1.1 x num_neg codes with randsubseq, which come
   out ascending, and keeps the first num_neg: the highest codes (sources with the largest ids) are almost never
   chosen.  Here every available code is equally likely to be in the sample.
3. No duplicate pairs.  Bidirected negatives are drawn as unordered pairs {a, b} and then mirrored, so the output has
   each pair once in each direction; the reference samples ordered codes and mirrors them, so (a, b) and (b, a) can
   both be drawn and appear twice.  The count is exact rather than "at most": min(num_neg, available).
4. perturb_edges' new edges are distinct from each other (they may still coincide with existing edges, as in the
   reference), and `max_trials` of negative_sample is accepted but unused: the result is exact, not trial-based.
5. Randomness comes from a `seed` keyword and is reproducible across GPUs; without one a seed is drawn from torch's
   default generator.  The reference takes a Julia `rng`.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Optional

import torch

from . import _lib
from . import graph as _graph
from ._lib import lib
from .basic import GNNLayer
from .graph import GNNGraph, _as_index, _stream
from .msgpass import apply_edges, xi_dot_xj
from .query import has_multi_edges, has_self_loops, is_bidirected

_SPACES = {(True, True): _lib.CODES_DIRECTED, (True, False): _lib.CODES_DIRECTED_NOLOOP,
           (False, True): _lib.CODES_UNDIRECTED, (False, False): _lib.CODES_UNDIRECTED_NOLOOP}


def space_size(space: int, n1: int, n2: Optional[int] = None) -> int:
    """M, the number of codes of a space (the reference's maxid)"""
    n1 = int(n1)
    return {_lib.CODES_DIRECTED: n1 * n1, _lib.CODES_DIRECTED_NOLOOP: n1 * (n1 - 1),
            _lib.CODES_UNDIRECTED: n1 * (n1 + 1) // 2, _lib.CODES_UNDIRECTED_NOLOOP: n1 * (n1 - 1) // 2,
            _lib.CODES_BIPARTITE: n1 * int(n2 or 0)}[space]


def _seed(seed) -> int:
    if seed is None:
        seed = int(torch.randint(0, 2 ** 62, (1,)).item())
    return int(seed) & (2 ** 64 - 1)


def _device(*ts) -> torch.device:
    for t in ts:
        if isinstance(t, torch.Tensor):
            return _graph._compute_device(t)
    return _graph._compute_device(torch.empty(0))


def _ids(v, dev) -> torch.Tensor:
    return _as_index(v).reshape(-1).to(device=dev, dtype=torch.int64).contiguous()


def _encode(space, n1, n2, s, t, dev) -> torch.Tensor:
    """0-based codes (int64) of 1-based (s, t)"""
    codes = torch.empty(s.numel(), dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        _lib.check(lib.gnnb_edge_encode(space, int(n1), int(n2), s.data_ptr(), t.data_ptr(), s.numel(), 1,
                                        codes.data_ptr(), _stream(dev)))
    return codes


def _decode(space, n1, n2, codes, dev):
    """1-based (s, t) of 0-based codes"""
    s = torch.empty(codes.numel(), dtype=torch.int64, device=dev)
    t = torch.empty_like(s)
    with torch.cuda.device(dev):
        _lib.check(lib.gnnb_edge_decode(space, int(n1), int(n2), codes.data_ptr(), codes.numel(), 1, s.data_ptr(),
                                        t.data_ptr(), _stream(dev)))
    return s, t


def _codes_sorted(space, n, s, t, dev) -> torch.Tensor:
    """the distinct codes of the pairs (s, t) the space holds, ascending"""
    out = torch.empty(s.numel(), dtype=torch.int64, device=dev)
    cnt = C.c_int64(0)
    with torch.cuda.device(dev):
        _lib.check(lib.gnnb_edge_codes_sorted(space, int(n), int(n), s.data_ptr(), t.data_ptr(), s.numel(), 1,
                                              out.data_ptr(), C.byref(cnt), _stream(dev)))
    return out[:int(cnt.value)]


def _member(codes, sorted_set, dev) -> torch.Tensor:
    flags = torch.empty(codes.numel(), dtype=torch.bool, device=dev)
    with torch.cuda.device(dev):
        _lib.check(lib.gnnb_codes_member(codes.data_ptr(), codes.numel(),
                                         sorted_set.data_ptr() if sorted_set.numel() else None, sorted_set.numel(),
                                         flags.data_ptr(), _stream(dev)))
    return flags


def sample_codes(M: int, m: int, *, exclude: Optional[torch.Tensor] = None, seed=None, device=None) -> torch.Tensor:
    """The first min(m, M - len(exclude)) codes of the seeded permutation π of [0, M) that are not in `exclude`
    (ascending distinct int64 codes), in π order — `gnnb_sample_codes`."""
    dev = torch.device(device) if device is not None else _device(exclude)
    excl = None if exclude is None else exclude.to(device=dev, dtype=torch.int64).contiguous()
    x = 0 if excl is None else int(excl.numel())
    out = torch.empty(max(0, min(int(m), int(M) - x)), dtype=torch.int64, device=dev)
    cnt = C.c_int64(0)
    with torch.cuda.device(dev):
        _lib.check(lib.gnnb_sample_codes(int(M), excl.data_ptr() if x else None, x, int(m), _seed(seed),
                                         out.data_ptr() if out.numel() else None, C.byref(cnt), _stream(dev)))
    return out[:int(cnt.value)]


# ---------------------------------------------------------------------------------------------- encoding / decoding
def edge_encoding(s, t, n: int, n2: Optional[int] = None, *, directed: bool = True, self_loops: bool = True):
    """(idx, maxid) with 1-based idx as in utils.jl:189-227; with n2 the bipartite code (s - 1) n2 + t.  Undirected
    pairs are encoded as (min, max); a self loop in a space without them is an AssertionError."""
    dev = _device(s, t)
    s, t = _ids(s, dev), _ids(t, dev)
    assert s.numel() == t.numel(), "s and t must have the same length"
    space = _lib.CODES_BIPARTITE if n2 is not None else _SPACES[(bool(directed), bool(self_loops))]
    return _encode(space, n, n if n2 is None else n2, s, t, dev) + 1, space_size(space, n, n2)


def edge_decoding(idx, n: int, n2: Optional[int] = None, *, directed: bool = True, self_loops: bool = True):
    """(s, t) of 1-based codes (utils.jl:229-268; `edge_decoding(idx, n1, n2)` for bipartite codes).  Exact for every
    n < 2^31; a code outside 1:maxid is an AssertionError."""
    dev = _device(idx)
    space = _lib.CODES_BIPARTITE if n2 is not None else _SPACES[(bool(directed), bool(self_loops))]
    codes = _ids(idx, dev) - 1
    return _decode(space, n, n if n2 is None else n2, codes, dev)


# ---------------------------------------------------------------------------------------------- graphs
def _dup_edata(edata, half: int):
    """bidirected rand_graph: edge features given for the m/2 drawn edges also go on their reverses"""
    if edata is None:
        return None
    d = {"e": edata} if isinstance(edata, torch.Tensor) else dict(edata)
    return {k: torch.cat([v, v], dim=-1) if v.shape[-1] == half else v for k, v in d.items()}


def rand_graph(n: int, m: int, *, bidirected: bool = True, edge_weight=None, seed=None, device=None,
               **kws) -> GNNGraph:
    """An Erdős–Rényi graph with n nodes and m distinct edges, no self loops (generate.jl:51-65).  Bidirected: m/2
    unordered pairs, each edge followed m/2 positions later by its reverse; edge_weight (length m/2) and edge
    features of m/2 columns are repeated for the reverses."""
    n, m = int(n), int(m)
    if bidirected:
        assert m % 2 == 0, f"Need even number of edges for bidirected graphs, given m={m}."
    space = _lib.CODES_UNDIRECTED_NOLOOP if bidirected else _lib.CODES_DIRECTED_NOLOOP
    k = m // 2 if bidirected else m
    M = space_size(space, n)
    assert 0 <= k <= M, f"{k} distinct edges asked of {n} nodes, which have {M}"
    dev = torch.device(device) if device is not None else _device()
    s, t = _decode(space, n, n, sample_codes(M, k, seed=seed, device=dev), dev)
    w = None
    if edge_weight is not None:
        w = torch.as_tensor(edge_weight, dtype=torch.float32).to(dev).reshape(-1)
    if bidirected:
        s, t = torch.cat([s, t]), torch.cat([t, s])
        w = None if w is None else torch.cat([w, w])
        if "edata" in kws:
            kws["edata"] = _dup_edata(kws["edata"], k)
    return GNNGraph(s, t, w, num_nodes=n, **kws)


def negative_sample(g: GNNGraph, *, max_trials: int = 3, num_neg_edges: Optional[int] = None,
                    bidirected: Optional[bool] = None, seed=None) -> GNNGraph:
    """min(num_neg_edges, available) random non-edges of g, as a graph on g's nodes (transform.jl:890-929).  Self loops
    are never negatives.  Bidirected: num_neg_edges ÷ 2 unordered pairs {a, b} that are not an edge of g in either
    direction, returned as [s; t] -> [t; s].  `max_trials` is accepted for compatibility and unused."""
    del max_trials
    assert g.num_graphs == 1, "negative_sample needs a single graph"
    n = g.num_nodes
    assert n >= 2, "negative_sample needs at least 2 nodes"
    num_neg = g.num_edges if num_neg_edges is None else int(num_neg_edges)
    assert num_neg >= 0, "num_neg_edges must be >= 0"
    if bidirected is None:
        bidirected = is_bidirected(g)
    dev = _device(g.s)
    s, t = _ids(g.s, dev), _ids(g.t, dev)
    space = _lib.CODES_UNDIRECTED_NOLOOP if bidirected else _lib.CODES_DIRECTED_NOLOOP
    positives = _codes_sorted(space, n, s, t, dev)
    codes = sample_codes(space_size(space, n), num_neg // 2 if bidirected else num_neg, exclude=positives, seed=seed,
                         device=dev)
    sn, tn = _decode(space, n, n, codes, dev)
    if bidirected:
        sn, tn = torch.cat([sn, tn]), torch.cat([tn, sn])
    return GNNGraph(sn, tn, num_nodes=n)


def rand_edge_split(g: GNNGraph, frac: float, *, bidirected: Optional[bool] = None, seed=None):
    """(g1, g2): a random round(ne · frac) of the edges and the rest (transform.jl:945-968), ne = E, or E/2 pairs when
    bidirected (an edge and its reverse go to the same side; the graph must then be bidirected, without self loops
    and without multi-edges)."""
    frac = float(frac)
    assert 0 <= frac <= 1, "frac must be between 0 and 1"
    if bidirected is None:
        bidirected = is_bidirected(g)
    dev = _device(g.s)
    s, t = g.s.to(dev), g.t.to(dev)
    if bidirected:
        assert is_bidirected(g), "rand_edge_split(bidirected=true) needs a bidirected graph"
        assert not has_self_loops(g), "rand_edge_split(bidirected=true) needs a graph without self loops"
        assert not has_multi_edges(g), "rand_edge_split(bidirected=true) needs a graph without multi-edges"
        mask = s < t
        s, t = s[mask], t[mask]
    ne = int(s.numel())
    eids = sample_codes(ne, ne, seed=seed, device=dev)
    size1 = round(ne * frac)
    e1, e2 = eids[:size1], eids[size1:]
    s1, t1, s2, t2 = s[e1], t[e1], s[e2], t[e2]
    if bidirected:
        s1, t1 = torch.cat([s1, t1]), torch.cat([t1, s1])
        s2, t2 = torch.cat([s2, t2]), torch.cat([t2, s2])
    return GNNGraph(s1, t1, num_nodes=g.num_nodes), GNNGraph(s2, t2, num_nodes=g.num_nodes)


def add_edges(g: GNNGraph, snew, tnew=None, *, edata=None) -> GNNGraph:
    """`add_edges(g, (s, t[, w]))` / `add_edges(g, s, t)` (transform.jl:319-353): the new edges after the old ones.
    Weights: missing ones on either side are padded with 1; edge features must come for the new edges under the same
    names; nodes beyond g.num_nodes are added (g must then have no node features)."""
    if tnew is None:
        data = tuple(snew)
        snew, tnew, wnew = data if len(data) == 3 else (data[0], data[1], None)
    else:
        wnew = None
    dev = g.s.device
    snew = _as_index(snew, dev).reshape(-1).to(g.s.dtype)
    tnew = _as_index(tnew, dev).reshape(-1).to(g.s.dtype)
    num_new = int(snew.numel())
    assert num_new == tnew.numel(), "s and t of the new edges must have the same length"
    assert wnew is None or len(wnew) == num_new, "one weight per new edge"
    if num_new == 0:
        return g
    assert int(snew.min()) >= 1 and int(tnew.min()) >= 1, "node ids are 1-based"
    new_ed = {} if edata is None else ({"e": edata} if isinstance(edata, torch.Tensor) else dict(edata))
    assert sorted(new_ed) == sorted(g.edata), "cannot concatenate feature data with different keys"
    ed = {k: torch.cat([v, torch.as_tensor(new_ed[k]).to(v.device, v.dtype)], dim=-1) for k, v in g.edata.items()}
    w = g.w
    if w is not None or wnew is not None:
        w_old = w if w is not None else torch.ones(g.num_edges, dtype=torch.float32, device=dev)
        w_new = torch.as_tensor(wnew, dtype=torch.float32).to(dev) if wnew is not None else \
            torch.ones(num_new, dtype=torch.float32, device=dev)
        w = torch.cat([w_old, w_new])
    n = max(int(snew.max()), int(tnew.max()), g.num_nodes)
    assert n == g.num_nodes or not g.ndata, "cannot add nodes to a graph with node features"
    return GNNGraph(torch.cat([g.s, snew]), torch.cat([g.t, tnew]), w, num_nodes=n, ndata=g.ndata, edata=ed,
                    gdata=g.gdata, num_graphs=g.num_graphs, graph_indicator=g.graph_indicator)


def perturb_edges(g: GNNGraph, perturb_ratio: float, *, seed=None) -> GNNGraph:
    """g plus ceil(E · perturb_ratio) random edges without self loops, distinct from each other, without weights or
    features of their own (transform.jl:385-418; add_edges pads the weights)."""
    perturb_ratio = float(perturb_ratio)
    assert 0 <= perturb_ratio <= 1, "perturb_ratio must be between 0 and 1"
    k = math.ceil(g.num_edges * perturb_ratio)
    if k == 0:
        return g
    n = g.num_nodes
    assert n > 1, "Graph must contain at least 2 nodes to add edges"
    M = space_size(_lib.CODES_DIRECTED_NOLOOP, n)
    assert k <= M, f"{k} new distinct edges asked of {n} nodes, which have {M}"
    dev = _device(g.s)
    s, t = _decode(_lib.CODES_DIRECTED_NOLOOP, n, n, sample_codes(M, k, seed=seed, device=dev), dev)
    return add_edges(g, (s.to(g.s.device), t.to(g.s.device)))


def _first_occurrences(s, t, n, dev) -> torch.Tensor:
    """mask of the edges that are the first of their (s, t) pair in COO order (the stable pair sort's run heads)"""
    E = int(s.numel())
    so, to = torch.empty_like(s), torch.empty_like(t)
    perm = torch.empty(E, dtype=torch.int64, device=dev)
    seg = torch.empty(E, dtype=torch.int64, device=dev)
    nu = C.c_int64(0)
    with torch.cuda.device(dev):
        _lib.check(lib.gnnb_coalesce_edges(s.data_ptr(), t.data_ptr(), E, int(n), 8, 1, so.data_ptr(), to.data_ptr(),
                                           perm.data_ptr(), seg.data_ptr(), C.byref(nu), _stream(dev)))
    head = torch.ones(E, dtype=torch.bool, device=dev)
    head[1:] = seg[1:] != seg[:-1]
    first = torch.zeros(E, dtype=torch.bool, device=dev)
    first[perm[head]] = True
    return first


def intersect(g1: GNNGraph, g2: GNNGraph) -> GNNGraph:
    """The edges of g1 that are also edges of g2, each pair once, in g1's order (operators.jl:7-20)."""
    assert g1.num_nodes == g2.num_nodes, "intersect needs graphs with the same number of nodes"
    n = g1.num_nodes
    dev = _device(g1.s)
    s1, t1, s2, t2 = _ids(g1.s, dev), _ids(g1.t, dev), _ids(g2.s, dev), _ids(g2.t, dev)
    if s1.numel() == 0 or s2.numel() == 0:
        return GNNGraph(s1[:0], t1[:0], num_nodes=n)
    codes1 = _encode(_lib.CODES_DIRECTED, n, n, s1, t1, dev)
    keep = _member(codes1, _codes_sorted(_lib.CODES_DIRECTED, n, s2, t2, dev), dev) & _first_occurrences(s1, t1, n, dev)
    return GNNGraph(s1[keep], t1[keep], num_nodes=n)


# ---------------------------------------------------------------------------------------------- decoder
def dot_decoder(g: GNNGraph, x: torch.Tensor) -> torch.Tensor:
    """(1, E) scores x_s · x_t — GNNlib/src/layers/basic.jl:1-3: apply_edges(xi_dot_xj, g, xi = x, xj = x)."""
    return apply_edges(xi_dot_xj, g, xi=x, xj=x)


class DotDecoder(GNNLayer):
    """DotDecoder() — GraphNeuralNetworks/src/layers/basic.jl:187-212; no parameters."""

    def forward(self, g: GNNGraph, x: torch.Tensor) -> torch.Tensor:
        return dot_decoder(g, x)
