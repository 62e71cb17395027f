"""Model composition — GraphNeuralNetworks/src/layers/basic.jl:

    GNNLayer    basic.jl:1-12     the base of every layer that takes the graph; l(g) = GNNGraph(g, ndata = l(g, x))
    WithGraph   basic.jl:14-52    a model tied to one graph: wg(x...) = model(g, x...)
    GNNChain    basic.jl:54-185   layers applied in sequence, the graph passed to the GNNLayers only
    Parallel    Flux.Parallel, as GNNChain applies it (basic.jl:158-166): connection(branch(x) for each branch)

Array layouts are the package's Julia-shaped ones (graph.py); nothing here touches the device.
"""
from __future__ import annotations

import numbers

import torch

from .graph import GNNGraph, edge_features, node_features


class GNNLayer(torch.nn.Module):
    """abstract type GNNLayer (basic.jl:1-12): a torch.nn.Module whose call with a lone GNNGraph is
    ``graph_forward(g)``, by default ``GNNGraph(g, ndata=self(g, node_features(g)))``.  Every other call is the Module's
    forward, unchanged."""

    def __call__(self, *args, **kw):
        if len(args) == 1 and not kw and isinstance(args[0], GNNGraph):
            return self.graph_forward(args[0])
        return super().__call__(*args, **kw)

    def graph_forward(self, g: GNNGraph) -> GNNGraph:
        return GNNGraph(g, ndata=self(g, node_features(g)))


class _EdgeFeatureLayer(GNNLayer):
    """the layers whose graph-only call also passes edge_features(g) (conv.jl:344, 464, 721, 936, 1140, 1540)"""

    def graph_forward(self, g: GNNGraph) -> GNNGraph:
        return GNNGraph(g, ndata=self(g, node_features(g), edge_features(g)))


class Parallel(torch.nn.Module):
    """Parallel(connection, *branches) — Flux.Parallel with one input: ``connection(*(b(x) for b in branches))``.
    Inside a GNNChain a branch that is a GNNLayer gets the graph too (basic.jl:158-166)."""

    def __init__(self, connection, *branches):
        super().__init__()
        if not branches:
            raise ValueError("Parallel needs at least one branch")
        self.connection = connection
        self.branches = tuple(branches)
        for i, b in enumerate(branches):
            if isinstance(b, torch.nn.Module):
                self.add_module(str(i), b)

    def forward(self, x):
        return self.connection(*(b(x) for b in self.branches))


def _applylayer(l, g: GNNGraph, x):
    """basic.jl:150-166: l(g, x) for a GNNLayer, l(x) for anything else"""
    if isinstance(l, Parallel):
        return l.connection(*(_applylayer(b, g, x) for b in l.branches))
    if isinstance(l, GNNLayer):
        return l(g, x)
    return l(x)


def _applylayer_graph(l, g: GNNGraph) -> GNNGraph:
    if isinstance(l, GNNLayer):
        return l(g)
    if isinstance(l, Parallel):
        return GNNGraph(g, ndata=_applylayer(l, g, node_features(g)))
    return GNNGraph(g, ndata=l(node_features(g)))


class GNNChain(GNNLayer):
    """GNNChain(*layers), GNNChain(list_of_layers) or GNNChain(**named_layers) — basic.jl:54-185.

    ``chain(g, x)`` passes x through the layers in order, calling ``l(g, x)`` on a GNNLayer and ``l(x)`` on anything
    else (a Module or a plain callable); ``chain(g)`` calls ``l(g)`` on a GNNLayer and otherwise replaces the node
    features by ``l(node_features(g))``.  ``len``, iteration, ``chain[i]``, ``chain["name"]``, and slices or lists of
    indices (which give a GNNChain of the same form) as the reference.  Module members are registered once each, so
    parameters(), train() and eval() reach all of them."""

    def __init__(self, *layers, **named):
        super().__init__()
        if layers and named:
            raise TypeError("GNNChain takes positional or named layers, not both")
        if "layers" in named:
            raise ValueError("a GNNChain cannot have a named layer called `layers`")
        if len(layers) == 1 and isinstance(layers[0], list):
            self._layers, self._names, self._vector = list(layers[0]), None, True
        elif named:
            self._layers, self._names, self._vector = list(named.values()), list(named), False
        else:
            self._layers, self._names, self._vector = list(layers), None, False
        for i, l in enumerate(self._layers):
            if isinstance(l, torch.nn.Module):
                self.add_module(str(i) if self._names is None else self._names[i], l)

    @property
    def layers(self):
        """the layers in order: a list for the vector form, a tuple otherwise"""
        return list(self._layers) if self._vector else tuple(self._layers)

    def keys(self):
        return list(self._names) if self._names is not None else list(range(len(self._layers)))

    def __len__(self):
        return len(self._layers)

    def __iter__(self):
        return iter(self._layers)

    def _sub(self, idx):
        if self._vector:
            return GNNChain([self._layers[i] for i in idx])
        if self._names is not None:
            return GNNChain(**{self._names[i]: self._layers[i] for i in idx})
        return GNNChain(*(self._layers[i] for i in idx))

    def __getitem__(self, i):
        if isinstance(i, str):
            if self._names is None or i not in self._names:
                raise KeyError(i)
            return self._layers[self._names.index(i)]
        if isinstance(i, slice):
            return self._sub(range(len(self._layers))[i])
        if isinstance(i, (list, tuple)):
            n = len(self._layers)
            return self._sub([range(n)[j] for j in i])
        if isinstance(i, numbers.Integral) and not isinstance(i, bool):
            return self._layers[i]
        raise TypeError(f"GNNChain indices are ints, names, slices or lists of ints (got {type(i).__name__})")

    def forward(self, g: GNNGraph, x):
        for l in self._layers:
            x = _applylayer(l, g, x)
        return x

    def graph_forward(self, g: GNNGraph) -> GNNGraph:
        for l in self._layers:
            g = _applylayer_graph(l, g)
        return g

    def __repr__(self):
        if self._names is not None:
            inner = ", ".join(f"{k} = {l!r}" for k, l in zip(self._names, self._layers))
        else:
            inner = ", ".join(repr(l) for l in self._layers)
            if self._vector:
                inner = f"[{inner}]"
        return f"GNNChain({inner})"


class WithGraph(torch.nn.Module):
    """WithGraph(model, g, traingraph=False) — basic.jl:14-52: ``wg(*x)`` is ``model(g, *x)`` and ``wg(g2, *x)`` is
    ``model(g2, *x)``.  Its parameters are the model's and, with traingraph=True, also the graph's floating arrays that
    require grad (the edge weight and the ndata / edata / gdata stores)."""

    def __init__(self, model, g: GNNGraph, traingraph: bool = False):
        super().__init__()
        self.model = model
        self.g = g
        self.traingraph = bool(traingraph)

    def forward(self, *args, **kw):
        if args and isinstance(args[0], GNNGraph):
            return self.model(*args, **kw)
        return self.model(self.g, *args, **kw)

    def _graph_arrays(self):
        g = self.g
        arrays = [("w", g.w)] + [(f"{store}.{k}", v) for store in ("ndata", "edata", "gdata")
                                 for k, v in getattr(g, store).items()]
        return [(f"g.{name}", v) for name, v in arrays
                if isinstance(v, torch.Tensor) and v.is_floating_point() and v.requires_grad]

    def named_parameters(self, prefix: str = "", recurse: bool = True, remove_duplicate: bool = True):
        seen = set()
        for name, p in super().named_parameters(prefix=prefix, recurse=recurse, remove_duplicate=remove_duplicate):
            seen.add(id(p))
            yield name, p
        if self.traingraph:
            for name, v in self._graph_arrays():
                if not (remove_duplicate and id(v) in seen):
                    seen.add(id(v))
                    yield (f"{prefix}.{name}" if prefix else name), v
