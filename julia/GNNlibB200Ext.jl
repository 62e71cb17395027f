# GNNlibB200Ext.jl — the Julia side of the drop-in: a GNNlib package extension that routes the message-passing hot
# path to libgnnb200.so (include/gnnb200.h) with `ccall`, in exactly the place where the reference's own CUDA
# extension *disables* its fast path (GNNlib/ext/GNNlibCUDAExt.jl:13-32).
#
# STATUS: source only.  Julia is not installed in the build image or on the GPU box (SURVEY.md §0.3), so this file
# has never been executed; the same entry points are exercised through the Python/ctypes mirror
# (graphneuralnetworks.jl_b200/) whose tests transcribe the reference's.  Registration a maintainer adds to
# GNNlib/Project.toml next to the existing lines (GNNlib/Project.toml:17-23):
#
#     [weakdeps]      CUDA, ChainRulesCore (already a dependency)
#     [extensions]    GNNlibB200Ext = "CUDA"          # same trigger as GNNlibCUDAExt
#
# and `ENV["GNNB200_LIB"]` (or a JLL) pointing at libgnnb200.so.
#
# Dispatch.  GNNlibCUDAExt's three methods are
#   propagate(::typeof(copy_xj|e_mul_xj|w_mul_xj), g::GNNGraph{<:Union{COO_T,SPARSE_T}}, ::typeof(+), xi, xj::AnyCuMatrix, e)
# Both extensions load on the CUDA trigger, and neither those nor the widened methods below (any fused aggregation, any
# rank of xj, Float32 only) are more specific than the other, so the headline call
# `propagate(copy_xj, coo_g, +, xi, ::CuMatrix{Float32}, e)` would be ambiguous.  The methods marked "intersection"
# below carry exactly the intersection signature (COO graph, `+`, CuMatrix{Float32}) and resolve it; a maintainer who
# prefers may instead delete the three methods of GNNlibCUDAExt (INTEGRATION.md says so too).
module GNNlibB200Ext

using CUDA
using ChainRulesCore
using Random
using Statistics: mean
using LinearAlgebra: I, inv, SingularException
using GNNlib: GNNlib, propagate, copy_xj, e_mul_xj, w_mul_xj, expand_srcdst, check_num_nodes
using GNNGraphs: GNNGraphs, GNNGraph, COO_T, edge_index, get_edge_weight, TemporalSnapshotsGNNGraph

const LIB = get(ENV, "GNNB200_LIB", "libgnnb200")

# ---- status -> the reference's exception types (include/gnnb200.h gnnb_status) ---------------------------------
@inline function check(st::Cint)
    st == 0 && return nothing
    msg = unsafe_string(ccall((:gnnb_last_error, LIB), Cstring, ()))
    (st == 2 || st == 6) && throw(AssertionError(msg))      # GNNB_ESIZE / GNNB_EINDEX  (GNNGraphs/src/utils.jl:1-28)
    st == 1 && throw(ArgumentError(msg))                    # GNNB_EINVAL               (GNNlib/src/layers/conv.jl:3-10)
    error("libgnnb200 status $st: $msg")
end

stream() = Base.unsafe_convert(Ptr{Cvoid}, CUDA.stream().handle)
cuptr(x::Nothing) = CU_NULL
cuptr(x) = pointer(x)

# ---- plan cache ----------------------------------------------------------------------------------------------------
# A graph is an immutable value `(s, t, num_nodes)`; its plan is found through the identity of BOTH index arrays plus the
# sizes.  The table is weak in `s` (a plan dies with the arrays it was built from: the finalizer frees the device CSR)
# and every entry checks `t` by identity through a WeakRef, so two graphs that share `s` but differ in `t` — a reversed
# or rewired graph, GNNGraph(s, t2) — get their own plans.
mutable struct Plan
    h::Ptr{Cvoid}
    loops::Union{Nothing, Plan}          # plan of add_self_loops(g), derived on first use (no second sort)
    function Plan(h)
        p = new(h, nothing)
        finalizer(p -> ccall((:gnnb_graph_destroy, LIB), Cint, (Ptr{Cvoid},), p.h), p)
    end
end
struct PlanEntry
    t::WeakRef
    num_nodes::Int
    num_edges::Int
    plan::Plan
end
const PLANS = WeakKeyDict{Any, Vector{PlanEntry}}()
const PLANS_LOCK = ReentrantLock()

function plan(g::GNNGraph{<:COO_T})
    s, t = edge_index(g)
    lock(PLANS_LOCK) do
        entries = get!(() -> PlanEntry[], PLANS, s)
        filter!(en -> en.t.value !== nothing, entries)
        for en in entries
            (en.t.value === t && en.num_nodes == g.num_nodes && en.num_edges == g.num_edges) && return en.plan
        end
        h = Ref{Ptr{Cvoid}}(C_NULL)
        check(ccall((:gnnb_graph_create, LIB), Cint,
                    (Ref{Ptr{Cvoid}}, CuPtr{Cvoid}, CuPtr{Cvoid}, Int64, Int64, Int64, Cint, Cint, Cint, Ptr{Cvoid}),
                    h, pointer(s), pointer(t), g.num_edges, g.num_nodes, g.num_nodes,
                    sizeof(eltype(s)), 1, 1, stream()))
        p = Plan(h[])
        push!(entries, PlanEntry(WeakRef(t), g.num_nodes, g.num_edges, p))
        return p
    end
end

# plan of add_self_loops(g) (GNNGraphs/src/transform.jl:12-28): loops appended after the originals
function loop_plan(p::Plan)
    p.loops === nothing || return p.loops
    h = Ref{Ptr{Cvoid}}(C_NULL)
    check(ccall((:gnnb_graph_add_self_loops, LIB), Cint, (Ptr{Cvoid}, Ref{Ptr{Cvoid}}, Ptr{Cvoid}), p.h, h, stream()))
    p.loops = Plan(h[])
end

const AGGR = IdDict{Any, Cint}(+ => 0, mean => 1, max => 2, min => 3)
const FusedAggr = Union{typeof(+), typeof(mean), typeof(max), typeof(min)}

# ---- the fused forward / pullback (gnnb_propagate, gnnb_propagate_bwd) ---------------------------------------------
function fused_propagate(p::Plan, aggr, xj::CuArray{Float32}, w::Union{Nothing, CuVector{Float32}})
    D = length(xj) ÷ size(xj)[end]
    out = similar(xj)
    check(ccall((:gnnb_propagate, LIB), Cint,
                (Ptr{Cvoid}, Cint, Cint, Cint, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, Int64,
                 CuPtr{Float32}, Ptr{Cvoid}),
                p.h, 0, w === nothing ? 0 : 1, AGGR[aggr], xj, cuptr(w), CU_NULL, CU_NULL, D, out, stream()))
    return out
end

function ChainRulesCore.rrule(::typeof(fused_propagate), p::Plan, aggr, xj, w)
    out = fused_propagate(p, aggr, xj, w)
    function fused_propagate_pullback(Δ)
        dout = CuArray{Float32}(unthunk(Δ))
        D = length(xj) ÷ size(xj)[end]
        dx = similar(xj)
        dw = w === nothing ? nothing : similar(w)
        check(ccall((:gnnb_propagate_bwd, LIB), Cint,
                    (Ptr{Cvoid}, Cint, Cint, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32},
                     CuPtr{Float32}, CuPtr{Float32}, Int64, CuPtr{Float32}, CuPtr{Float32}, Ptr{Cvoid}),
                    p.h, w === nothing ? 0 : 1, AGGR[aggr], dout, xj, cuptr(w), CU_NULL, CU_NULL, out, D, dx, cuptr(dw),
                    stream()))
        return NoTangent(), NoTangent(), NoTangent(), dx, dw === nothing ? NoTangent() : dw
    end
    return out, fused_propagate_pullback
end

## COPY_XJ — replaces GNNlib/ext/GNNlibCUDAExt.jl:13-16 (and adds mean/max/min, 3-D xj)
GNNlib.propagate(::typeof(copy_xj), g::GNNGraph{<:COO_T}, aggr::FusedAggr, xi, xj::CuArray{Float32}, e) =
    fused_propagate(plan(g), aggr, xj, nothing)
GNNlib.propagate(::typeof(copy_xj), g::GNNGraph{<:COO_T}, ::typeof(+), xi, xj::CuMatrix{Float32}, e) =   # intersection
    fused_propagate(plan(g), +, xj, nothing)

## E_MUL_XJ with a vector of edge weights — replaces GNNlibCUDAExt.jl:21-24
GNNlib.propagate(::typeof(e_mul_xj), g::GNNGraph{<:COO_T}, aggr::FusedAggr, xi, xj::CuArray{Float32},
                 e::CuVector{Float32}) = fused_propagate(plan(g), aggr, xj, e)
GNNlib.propagate(::typeof(e_mul_xj), g::GNNGraph{<:COO_T}, ::typeof(+), xi, xj::CuMatrix{Float32},         # intersection
                 e::CuVector{Float32}) = fused_propagate(plan(g), +, xj, e)

## W_MUL_XJ with the graph's own weights — replaces GNNlibCUDAExt.jl:29-32
GNNlib.propagate(::typeof(w_mul_xj), g::GNNGraph{<:COO_T}, aggr::FusedAggr, xi, xj::CuArray{Float32}, e::Nothing) =
    fused_propagate(plan(g), aggr, xj, get_edge_weight(g))
GNNlib.propagate(::typeof(w_mul_xj), g::GNNGraph{<:COO_T}, ::typeof(+), xi, xj::CuMatrix{Float32}, e::Nothing) =   # intersection
    fused_propagate(plan(g), +, xj, get_edge_weight(g))

## softmax_edge_neighbors — replaces GNNlib/src/utils.jl:84-97 on CuArrays
function GNNlib.softmax_edge_neighbors(g::GNNGraph{<:COO_T}, e::CuArray{Float32})
    @assert size(e)[end] == g.num_edges
    K = length(e) ÷ g.num_edges
    out = similar(e)
    check(ccall((:gnnb_softmax_edge_neighbors, LIB), Cint,
                (Ptr{Cvoid}, CuPtr{Float32}, Int64, CuPtr{Float32}, Ptr{Cvoid}), plan(g).h, e, K, out, stream()))
    return out
end

function ChainRulesCore.rrule(::typeof(GNNlib.softmax_edge_neighbors), g::GNNGraph{<:COO_T}, e::CuArray{Float32})
    α = GNNlib.softmax_edge_neighbors(g, e)
    function softmax_pullback(Δ)
        dα = CuArray{Float32}(unthunk(Δ))
        de = similar(e)
        check(ccall((:gnnb_softmax_edge_neighbors_bwd, LIB), Cint,
                    (Ptr{Cvoid}, CuPtr{Float32}, CuPtr{Float32}, Int64, CuPtr{Float32}, Ptr{Cvoid}),
                    plan(g).h, α, dα, length(e) ÷ g.num_edges, de, stream()))
        return NoTangent(), NoTangent(), de
    end
    return α, softmax_pullback
end

# ---- dense part of a layer: σ.(W * x .+ b) for σ ∈ {identity, relu} (gnnb_linear, gnnb_linear_bwd) -------------------
isrelu(σ) = nameof(σ) === :relu
fusable_σ(σ) = σ === identity || isrelu(σ)

function fused_linear(W::CuMatrix{Float32}, x::CuMatrix{Float32}, b::Union{Nothing, CuVector{Float32}}, relu::Bool)
    Dout, Din = size(W)
    N = size(x, 2)
    # the C entry takes W as the layer stores it in row-major (Dout, Din) terms = Julia's permuted copy
    Wr = permutedims(W)                                  # (Din, Dout) column-major == (Dout, Din) row-major
    y = similar(x, Dout, N)
    check(ccall((:gnnb_linear, LIB), Cint,
                (CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, Cint, Int64, Int64, Int64, CuPtr{Float32}, Ptr{Cvoid}),
                x, Wr, cuptr(b), relu, N, Din, Dout, y, stream()))
    return y
end

# relu(W * x .+ b) with its relu mask kept as bits (4 words per node) for the pullback; `nothing` when
# gnnb_linear_relu_mask does not serve the shape (Dout != 128, Din not 32, 64, 96 or 128)
function fused_linear_relu_mask(W::CuMatrix{Float32}, x::CuMatrix{Float32}, b::Union{Nothing, CuVector{Float32}})
    Dout, Din = size(W)
    N = size(x, 2)
    Wr = permutedims(W)
    y = similar(x, Dout, N)
    mask = CuArray{UInt32}(undef, 4, N)
    st = ccall((:gnnb_linear_relu_mask, LIB), Cint,
               (CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, Int64, Int64, Int64, CuPtr{Float32}, CuPtr{UInt32}, Ptr{Cvoid}),
               x, Wr, cuptr(b), N, Din, Dout, y, mask, stream())
    st == 5 && return nothing                            # GNNB_EUNSUPPORTED
    check(st)
    return y, mask
end

function ChainRulesCore.rrule(::typeof(fused_linear), W, x, b, relu::Bool)
    ym = relu ? fused_linear_relu_mask(W, x, b) : nothing
    if ym !== nothing
        y, mask = ym
        function fused_linear_mask_pullback(Δ)
            dy = CuArray{Float32}(unthunk(Δ))
            Dout, Din = size(W)
            N = size(x, 2)
            Wr = permutedims(W)
            dx, dWr = similar(x), similar(Wr)
            db = b === nothing ? nothing : similar(b)
            check(ccall((:gnnb_linear_bwd_mask, LIB), Cint,
                        (CuPtr{Float32}, CuPtr{UInt32}, CuPtr{Float32}, CuPtr{Float32}, Int64, Int64, Int64,
                         CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, Ptr{Cvoid}),
                        dy, mask, x, Wr, N, Din, Dout, dx, dWr, cuptr(db), stream()))
            return NoTangent(), permutedims(dWr), dx, db === nothing ? NoTangent() : db, NoTangent()
        end
        return y, fused_linear_mask_pullback
    end
    y = fused_linear(W, x, b, relu)
    function fused_linear_pullback(Δ)
        dy = CuArray{Float32}(unthunk(Δ))
        Dout, Din = size(W)
        N = size(x, 2)
        Wr = permutedims(W)
        dx, dWr = similar(x), similar(Wr)
        db = b === nothing ? nothing : similar(b)
        ws = relu ? similar(dy) : nothing
        check(ccall((:gnnb_linear_bwd, LIB), Cint,
                    (CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, Cint, Int64, Int64, Int64,
                     CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, Ptr{Cvoid}),
                    dy, relu ? pointer(y) : CU_NULL, x, Wr, relu, N, Din, Dout, cuptr(ws), dx, dWr, cuptr(db), stream()))
        return NoTangent(), permutedims(dWr), dx, db === nothing ? NoTangent() : db, NoTangent()
    end
    return y, fused_linear_pullback
end

# ---- closing line of a layer that ends in an aggregation: σ.(x .+ b) (gnnb_bias_act, gnnb_bias_act_bwd) ---------------
# one pass forward, one pass backward (mask product + deterministic bias gradient) instead of four broadcasts
function bias_act(x::CuMatrix{Float32}, b::Union{Nothing, CuVector{Float32}}, relu::Bool)
    D, N = size(x)
    y = similar(x)
    check(ccall((:gnnb_bias_act, LIB), Cint,
                (CuPtr{Float32}, CuPtr{Float32}, Cint, Int64, Int64, CuPtr{Float32}, Ptr{Cvoid}),
                x, cuptr(b), relu, N, D, y, stream()))
    return y
end

function ChainRulesCore.rrule(::typeof(bias_act), x, b, relu::Bool)
    y = bias_act(x, b, relu)
    function bias_act_pullback(Δ)
        dy = CuArray{Float32}(unthunk(Δ))
        D, N = size(dy)
        dpre = relu ? similar(dy) : dy
        db = b === nothing ? nothing : similar(b)
        (relu || db !== nothing) &&
            check(ccall((:gnnb_bias_act_bwd, LIB), Cint,
                        (CuPtr{Float32}, CuPtr{Float32}, Cint, Int64, Int64, CuPtr{Float32}, CuPtr{Float32}, Ptr{Cvoid}),
                        dy, relu ? pointer(y) : CU_NULL, relu, N, D, relu ? pointer(dpre) : CU_NULL, cuptr(db), stream()))
        return NoTangent(), dpre, db === nothing ? NoTangent() : db, NoTangent()
    end
    return y, bias_act_pullback
end

closing(l, y::CuMatrix{Float32}) =
    (fusable_σ(l.σ) && size(y, 1) % 4 == 0 && size(y, 1) <= 1024 && (l.bias === false || l.bias isa CuVector{Float32})) ?
    bias_act(y, l.bias === false ? nothing : l.bias, isrelu(l.σ)) : l.σ.(y .+ l.bias)

dense(l, W, x, with_bias_act::Bool) = begin
    b = (with_bias_act && l.bias isa CuVector{Float32}) ? l.bias : nothing
    σ = with_bias_act ? l.σ : identity
    if fusable_σ(σ) && size(W, 1) % 4 == 0 && size(W, 2) % 4 == 0 && (l.bias === false || l.bias isa CuVector{Float32} || !with_bias_act)
        fused_linear(W, x, b, isrelu(σ))
    else
        with_bias_act ? σ.(W * x .+ l.bias) : W * x
    end
end

# ---- gcn_conv fast path (GNNlib/src/layers/conv.jl:14-72; callers GraphNeuralNetworks/src/layers/conv.jl:103, GNNLux :137)
# c .* propagate(copy_xj | e_mul_xj, g', +, xj = x .* c') in ONE pass over the self-loop plan, both scalings folded into the
# gather and the store (gnnb_gcn_propagate), and its pullback (the same kernel on the CSR-by-source plan).
function gcn_core(p::Plan, x::CuMatrix{Float32}, c::CuVector{Float32})
    out = similar(x)
    check(ccall((:gnnb_gcn_propagate, LIB), Cint,
                (Ptr{Cvoid}, Cint, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, Int64, CuPtr{Float32}, Ptr{Cvoid}),
                p.h, 0, x, CU_NULL, c, size(x, 1), out, stream()))
    return out
end
function ChainRulesCore.rrule(::typeof(gcn_core), p::Plan, x, c)
    out = gcn_core(p, x, c)
    function gcn_core_pullback(Δ)
        dout = CuArray{Float32}(unthunk(Δ))
        dx = similar(x)
        check(ccall((:gnnb_gcn_propagate, LIB), Cint,
                    (Ptr{Cvoid}, Cint, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, Int64, CuPtr{Float32}, Ptr{Cvoid}),
                    p.h, 1, dout, CU_NULL, c, size(x, 1), dx, stream()))
        return NoTangent(), NoTangent(), dx, NoTangent()       # c is a function of the graph only (unweighted)
    end
    return out, gcn_core_pullback
end

# gcn_conv on a one-relation GNNHeteroGraph (GNNlib/src/layers/conv.jl:45-50,58-66): sources scaled by 1/sqrt(out-degree),
# targets by 1/sqrt(in-degree), on the relation's bipartite plan (gnnb_gcn_propagate_bipartite).  x is (D, num_src), the
# result (D, num_dst); the pullback is the same entry with transposed = 1.
function gcn_core_bipartite(p::Plan, x::CuMatrix{Float32}, n_dst::Integer)
    out = CuMatrix{Float32}(undef, size(x, 1), n_dst)
    check(ccall((:gnnb_gcn_propagate_bipartite, LIB), Cint,
                (Ptr{Cvoid}, Cint, CuPtr{Float32}, Int64, CuPtr{Float32}, Ptr{Cvoid}),
                p.h, 0, x, size(x, 1), out, stream()))
    return out
end
function ChainRulesCore.rrule(::typeof(gcn_core_bipartite), p::Plan, x, n_dst)
    out = gcn_core_bipartite(p, x, n_dst)
    function gcn_core_bipartite_pullback(Δ)
        dout = CuArray{Float32}(unthunk(Δ))
        dx = similar(x)
        check(ccall((:gnnb_gcn_propagate_bipartite, LIB), Cint,
                    (Ptr{Cvoid}, Cint, CuPtr{Float32}, Int64, CuPtr{Float32}, Ptr{Cvoid}),
                    p.h, 1, dout, size(x, 1), dx, stream()))
        return NoTangent(), NoTangent(), dx, NoTangent()       # the scales depend on the graph only (unweighted)
    end
    return out, gcn_core_bipartite_pullback
end

function in_degree(p::Plan, n::Integer)
    d = CUDA.zeros(Float32, n)
    check(ccall((:gnnb_degree, LIB), Cint, (Ptr{Cvoid}, Cint, CuPtr{Float32}, CuPtr{Float32}, Ptr{Cvoid}),
                p.h, 1, CU_NULL, d, stream()))
    return d
end
ChainRulesCore.@non_differentiable in_degree(::Any...)
ChainRulesCore.@non_differentiable plan(::Any...)
ChainRulesCore.@non_differentiable loop_plan(::Any...)

function GNNlib.gcn_conv(l, g::GNNGraph{<:COO_T}, x::CuMatrix{Float32}, edge_weight::Nothing, norm_fn::F,
                         conv_weight::Union{Nothing, CuMatrix{Float32}}) where {F}
    (l.use_edge_weight && get_edge_weight(g) !== nothing) &&            # weighted graphs: the reference's own body, whose
        return invoke(GNNlib.gcn_conv, Tuple{Any, GNNlib.AbstractGNNGraph, Any, Nothing, F, typeof(conv_weight)},
                      l, g, x, edge_weight, norm_fn, conv_weight)      # propagate calls reach the fused methods above
    weight = conv_weight === nothing ? l.weight : conv_weight
    size(weight) == size(l.weight) ||
        throw(ArgumentError("The weight matrix has the wrong size. Expected $(size(l.weight)) but got $(size(weight))"))
    check_num_nodes(g, x)
    Dout, Din = size(weight)
    p = l.add_self_loops ? loop_plan(plan(g)) : plan(g)
    Dout < Din && (x = dense(l, weight, x, false))                       # multiply before convolution (conv.jl:36-40)
    c = norm_fn(in_degree(p, g.num_nodes))                               # conv.jl:52-57, any norm_fn
    x = gcn_core(p, x, c)
    Dout >= Din && return dense(l, weight, x, true)                      # σ.(W * x .+ b), bias/relu in the GEMM epilogue
    return l.σ.(x .+ l.bias)
end

# ---- gat_conv fast path (GNNlib/src/layers/conv.jl:112-167; callers GraphNeuralNetworks/src/layers/conv.jl:346) ------
# logits -> leakyrelu -> neighbourhood softmax -> α-weighted sum of Wx rows in one pass (gnnb_gat_aggregate), no (C,H,E)
# tensors; the pullback recomputes α from the per-target statistics (gnnb_gat_aggregate_bwd).
function gat_aggregate(p::Plan, Wx::CuArray{Float32, 3}, el::CuMatrix{Float32}, er::CuMatrix{Float32}, slope::Float32)
    C, H, N = size(Wx)
    out = similar(Wx)
    check(ccall((:gnnb_gat_aggregate, LIB), Cint,
                (Ptr{Cvoid}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, Int64, Int64, Cfloat, CuPtr{Float32},
                 CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, Ptr{Cvoid}),
                p.h, Wx, el, er, C, H, slope, out, CU_NULL, CU_NULL, CU_NULL, stream()))
    return out
end
function ChainRulesCore.rrule(::typeof(gat_aggregate), p::Plan, Wx, el, er, slope)
    C, H, N = size(Wx)
    out = similar(Wx)
    smax, ssum = similar(el), similar(el)
    check(ccall((:gnnb_gat_aggregate, LIB), Cint,
                (Ptr{Cvoid}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, Int64, Int64, Cfloat, CuPtr{Float32},
                 CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, Ptr{Cvoid}),
                p.h, Wx, el, er, C, H, slope, out, CU_NULL, smax, ssum, stream()))
    function gat_aggregate_pullback(Δ)
        dout = CuArray{Float32}(unthunk(Δ))
        dWx, del, der = similar(Wx), similar(el), similar(er)
        check(ccall((:gnnb_gat_aggregate_bwd, LIB), Cint,
                    (Ptr{Cvoid}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32},
                     CuPtr{Float32}, CuPtr{Float32}, Int64, Int64, Cfloat, CuPtr{Float32}, CuPtr{Float32},
                     CuPtr{Float32}, Ptr{Cvoid}),
                    p.h, Wx, el, er, smax, ssum, out, dout, C, H, slope, dWx, del, der, stream()))
        return NoTangent(), NoTangent(), dWx, del, der, NoTangent()
    end
    return out, gat_aggregate_pullback
end

function GNNlib.gat_conv(l, g::GNNGraph{<:COO_T}, x::CuMatrix{Float32}, e::Nothing = nothing)
    (l.dense_e === nothing && iszero(l.dropout)) ||                      # edge features / dropout: the reference's body
        return invoke(GNNlib.gat_conv, Tuple{Any, GNNlib.AbstractGNNGraph, Any, Nothing}, l, g, x, e)
    check_num_nodes(g, x)
    p = l.add_self_loops ? loop_plan(plan(g)) : plan(g)
    _, chout = l.channel
    heads = l.heads
    Wx = reshape(l.dense_x(x), chout, heads, :)                          # conv.jl:128-129 (Dense without bias, :336)
    ai, aj = l.a[1:chout, :], l.a[(chout + 1):(2chout), :]               # rows 1..C pair with the target, C+1..2C with the source (:157)
    el = dropdims(sum(reshape(ai, chout, heads, 1) .* Wx, dims = 1), dims = 1)    # (H, N)
    er = dropdims(sum(reshape(aj, chout, heads, 1) .* Wx, dims = 1), dims = 1)
    y = gat_aggregate(p, Wx, el, er, Float32(l.negative_slope))
    l.concat || (y = mean(y, dims = 2))
    y = reshape(y, :, size(y, 3))
    return closing(l, y)                                                 # conv.jl:149, one pass
end

# ---- sage_conv fast path (GNNlib/src/layers/conv.jl:277-283; caller GraphNeuralNetworks/src/layers/conv.jl:787) ------
# σ.(W * [x_i ; m_i] .+ b) without the (2D, N) vcat temporary: the two column blocks of W hit x and m separately.
function GNNlib.sage_conv(l, g::GNNGraph{<:COO_T}, x::CuMatrix{Float32})
    check_num_nodes(g, x)
    xj, xi = expand_srcdst(g, x)
    m = propagate(copy_xj, g, l.aggr, xj = xj)                           # the fused mean / sum / max kernel
    Din = size(xi, 1)
    W1, W2 = l.weight[:, 1:Din], l.weight[:, (Din + 1):end]
    return l.σ.(W1 * xi .+ W2 * m .+ l.bias)
end

## sort_edge_index on device arrays — replaces GNNGraphs/ext/GNNGraphsCUDAExt.jl:24-30 (copy to the CPU, sort, copy back)
function GNNGraphs.sort_edge_index(u::CuVector{T}, v::CuVector{T}) where {T <: Union{Int32, Int64}}
    @assert length(u) == length(v)
    uo, vo = similar(u), similar(v)
    isempty(u) && return uo, vo
    hi = max(maximum(u), maximum(v))
    check(ccall((:gnnb_sort_edge_index, LIB), Cint,
                (CuPtr{T}, CuPtr{T}, Int64, Int64, Cint, CuPtr{T}, CuPtr{T}, CuPtr{Int64}, Ptr{Cvoid}),
                u, v, length(u), hi, sizeof(T), uo, vo, CU_NULL, stream()))
    return uo, vo
end

## remove_multi_edges on a device COO graph — the index half of GNNGraphs/src/transform.jl:157-190 in one call; the
## `_scatter(aggr, ·, idxs)` of the weights / edge features stays the reference's own line (NNlib.scatter on CuArrays).
function coalesce_edge_index(s::CuVector{T}, t::CuVector{T}, n::Integer) where {T <: Union{Int32, Int64}}
    E = length(s)
    so, to = similar(s), similar(t)
    perm, idxs = CUDA.zeros(Int64, E), CUDA.zeros(Int64, E)
    nu = Ref{Int64}(0)
    check(ccall((:gnnb_coalesce_edges, LIB), Cint,
                (CuPtr{T}, CuPtr{T}, Int64, Int64, Cint, Cint, CuPtr{T}, CuPtr{T}, CuPtr{Int64}, CuPtr{Int64},
                 Ref{Int64}, Ptr{Cvoid}),
                s, t, E, n, sizeof(T), 1, so, to, perm, idxs, nu, stream()))
    return so[1:nu[]], to[1:nu[]], perm .+ 1, idxs          # 1-based permutation, segment id of every sorted edge
end

## knn_graph / radius_graph on device points — replace GNNGraphs/src/generate.jl:112-145,196-222 (KDTree / BallTree on
## the CPU).  Exact fp32 distances within each graph of the batch; rows in (d2, j) order (knn) or ascending j (radius).
## The indicator is sorted on the device when it is not already non-decreasing, and the rows are mapped back; every step
## below stays on the device (no scalar indexing, no host copy of the neighbour lists).
function _knn_segments(graph_indicator, n)
    graph_indicator === nothing && return nothing, nothing, nothing
    @assert graph_indicator isa AbstractVector{<:Integer}
    @assert length(graph_indicator) == n
    gi = CuVector{Int64}(graph_indicator)
    n == 0 && return nothing, nothing, nothing
    order = nothing
    if !all(gi[2:end] .>= gi[1:end-1])
        # unique keys (graph, position): the sort is stable whatever algorithm sortperm picks
        keys = (gi .- minimum(gi)) .* Int64(n) .+ CuVector{Int64}(0:n-1)
        order = sortperm(keys)
    end
    gs = order === nothing ? gi : gi[order]
    ends = findall(gs[1:end-1] .!= gs[2:end])                 # last position of every graph but the last
    seg = vcat(CUDA.zeros(Int64, 1), Int64.(ends), CuVector{Int64}([n]))
    inv = nothing
    if order !== nothing
        inv = similar(order)
        inv[order] .= CuVector{Int64}(1:n)                    # sorted position of each node
    end
    return order, inv, seg
end

_knn_seg_args(seg) = seg === nothing ? (CU_NULL, 1) : (seg, length(seg) - 1)

function _knn_coo(centre, nbr, dir)
    @assert dir ∈ (:in, :out)
    return dir == :in ? (nbr, centre) : (centre, nbr)
end

# centre of every entry of a ragged list with `counts` entries per row (1-based rows), on the device: a +delta at the
# first entry of every non-empty row, then a running sum
function _ragged_centres(counts::CuVector{Int64}, total::Integer)
    centre = CUDA.zeros(Int64, total)
    total == 0 && return centre
    nz = findall(counts .> 0)
    nzv = Int64.(nz)
    starts = cumsum(counts)[nz] .- counts[nz] .+ 1
    centre[starts] .= nzv .- vcat(CUDA.zeros(Int64, 1), nzv[1:end-1])
    return cumsum(centre)
end

function GNNGraphs.knn_graph(points::CuMatrix{Float32}, k::Int; graph_indicator = nothing, self_loops = false,
                             dir = :in, kws...)
    @assert dir ∈ (:in, :out)
    d, n = size(points)
    order, inv, seg = _knn_segments(graph_indicator, n)
    x = order === nothing ? points : points[:, order]
    sp, ns = _knn_seg_args(seg)
    nbr = CuMatrix{Int32}(undef, k, n)                        # column i = row i of the C layout
    check(ccall((:gnnb_knn, LIB), Cint,
                (CuPtr{Float32}, Int64, Cint, CuPtr{Int64}, Int64, Cint, Cint, CuPtr{Int32}, Ptr{Cvoid}),
                x, n, d, sp, ns, k, self_loops, nbr, stream()))
    ids = Int64.(nbr) .+ 1
    if order !== nothing
        ids = order[ids[:, inv]]                              # columns back in node order, ids back to node ids
    end
    s, t = _knn_coo(repeat(CuVector{Int64}(1:n), inner = k), vec(ids), dir)
    return GNNGraph((s, t); num_nodes = n, graph_indicator, kws...)
end

function GNNGraphs.radius_graph(points::CuMatrix{Float32}, r::AbstractFloat; graph_indicator = nothing,
                                self_loops = false, dir = :in, kws...)
    @assert dir ∈ (:in, :out)
    d, n = size(points)
    order, inv, seg = _knn_segments(graph_indicator, n)
    x = order === nothing ? points : points[:, order]
    sp, ns = _knn_seg_args(seg)
    offsets = CUDA.zeros(Int64, n + 1)
    total = Ref{Int64}(0)
    check(ccall((:gnnb_radius_count, LIB), Cint,
                (CuPtr{Float32}, Int64, Cint, CuPtr{Int64}, Int64, Cfloat, Cint, CuPtr{Int64}, Ref{Int64}, Ptr{Cvoid}),
                x, n, d, sp, ns, r, self_loops, offsets, total, stream()))
    E = total[]
    nbr = CuVector{Int32}(undef, E)
    E > 0 && check(ccall((:gnnb_radius_fill, LIB), Cint,
                         (CuPtr{Float32}, Int64, Cint, CuPtr{Int64}, Int64, Cfloat, Cint, CuPtr{Int64}, CuPtr{Int32},
                          Int64, Ptr{Cvoid}),
                         x, n, d, sp, ns, r, self_loops, offsets, nbr, E, stream()))
    ids = Int64.(nbr) .+ 1
    counts = offsets[2:end] .- offsets[1:end-1]               # row lengths in sorted order
    if order === nothing
        centre = _ragged_centres(counts, E)
    else
        counts_out = counts[inv]                              # row lengths in node order
        centre = _ragged_centres(counts_out, E)
        start_out = cumsum(counts_out) .- counts_out          # 0-based start of each output row
        pos = CuVector{Int64}(0:E-1) .- start_out[centre]     # position inside the row
        src = offsets[1:end-1][inv][centre] .+ pos .+ 1       # the same entry in the sorted rows
        ids = order[ids[src]]
    end
    s, t = _knn_coo(centre, ids, dir)
    return GNNGraph((s, t); num_nodes = n, graph_indicator, kws...)
end

## rand_temporal_radius_graph / rand_temporal_hyperbolic_graph on the device — replace GNNGraphs/src/generate.jl:265-284
## (a BallTree per snapshot) and :287-297,340-380 (a dense n x n Float64 adjacency per snapshot).  Own names, so that
## GNNGraphs' array-free methods stay the CPU ones: the node dynamics of all T snapshots run in one launch from the seeded
## stream of include/gnnb200.h, then every snapshot's edges come from one count and one fill over the T snapshots as T
## segments.  One read-back of the T + 1 snapshot edge offsets; snapshot t is a slice of the flat rows.
function _temporal_snapshots(offsets::CuVector{Int64}, nbr::CuVector{Int32}, n, T, dir, weighted, kws)
    E = length(nbr)
    counts = offsets[2:end] .- offsets[1:end-1]
    centre = _ragged_centres(counts, E)                       # 1-based flat rows
    eoff = Array(offsets[(0:T) .* n .+ 1])
    snaps = Vector{GNNGraph}(undef, T)
    for t in 1:T
        a, b = eoff[t] + 1, eoff[t + 1]
        sh = (t - 1) * n
        s, d = _knn_coo(centre[a:b] .- sh, Int64.(nbr[a:b]) .+ (1 - sh), dir)
        snaps[t] = weighted ? GNNGraph((s, d, CUDA.ones(Float32, b - a + 1)); num_nodes = n, kws...) :
                              GNNGraph((s, d); num_nodes = n, kws...)
    end
    return TemporalSnapshotsGNNGraph(snaps)
end

function rand_temporal_radius_graph_cuda(n::Int, T::Int, speed::AbstractFloat, r::AbstractFloat; self_loops = false,
                                         dir = :in, seed = nothing, rng = Random.default_rng(), kws...)
    @assert dir ∈ (:in, :out)
    N = n * T
    pts = CuMatrix{Float32}(undef, 2, N)
    check(ccall((:gnnb_temporal_radius_points, LIB), Cint, (Int64, Int64, Cdouble, UInt64, CuPtr{Float32}, Ptr{Cvoid}),
                n, T, speed, _seed(rng, seed), pts, stream()))
    seg = CuVector{Int64}((0:T) .* n)
    offsets = CUDA.zeros(Int64, N + 1)
    total = Ref{Int64}(0)
    check(ccall((:gnnb_radius_count, LIB), Cint,
                (CuPtr{Float32}, Int64, Cint, CuPtr{Int64}, Int64, Cfloat, Cint, CuPtr{Int64}, Ref{Int64}, Ptr{Cvoid}),
                pts, N, 2, seg, T, r, self_loops, offsets, total, stream()))
    nbr = CuVector{Int32}(undef, total[])
    total[] > 0 && check(ccall((:gnnb_radius_fill, LIB), Cint,
                               (CuPtr{Float32}, Int64, Cint, CuPtr{Int64}, Int64, Cfloat, Cint, CuPtr{Int64}, CuPtr{Int32},
                                Int64, Ptr{Cvoid}),
                               pts, N, 2, seg, T, r, self_loops, offsets, nbr, total[], stream()))
    return _temporal_snapshots(offsets, nbr, n, T, dir, false, kws)
end

function rand_temporal_hyperbolic_graph_cuda(n::Int, T::Int; α::Real, R::Real, speed::Real, ζ::Real = 1,
                                             self_loop = false, seed = nothing, rng = Random.default_rng(), kws...)
    @assert T > 1 "The number of snapshots must be greater than 1"
    @assert α > 0 "α must be greater than 0"
    ζ > 0 && R >= 0 && all(isfinite, (α, R, speed, ζ)) && isfinite(cosh(α * R)) && isfinite(cosh(ζ * R)) ||
        throw(ArgumentError("need ζ > 0, R >= 0, finite parameters and finite cosh(αR), cosh(ζR)"))
    N = n * T
    rec = CuMatrix{Float64}(undef, 4, N)                      # column = the record (cosh ζr, sinh ζr, cos θ, sin θ)
    check(ccall((:gnnb_temporal_hyperbolic_records, LIB), Cint,
                (Int64, Int64, Cdouble, Cdouble, Cdouble, Cdouble, UInt64, CuPtr{Float64}, Ptr{Cvoid}),
                n, T, α, R, speed, ζ, _seed(rng, seed), rec, stream()))
    seg = CuVector{Int64}((0:T) .* n)
    offsets = CUDA.zeros(Int64, N + 1)
    total = Ref{Int64}(0)
    x_max = cosh(Float64(ζ) * R)                              # acosh(x)/ζ <= R without an acosh per pair
    check(ccall((:gnnb_hyperbolic_count, LIB), Cint,
                (CuPtr{Float64}, Int64, CuPtr{Int64}, Int64, Cdouble, Cint, CuPtr{Int64}, Ref{Int64}, Ptr{Cvoid}),
                rec, N, seg, T, x_max, self_loop, offsets, total, stream()))
    nbr = CuVector{Int32}(undef, total[])
    total[] > 0 && check(ccall((:gnnb_hyperbolic_fill, LIB), Cint,
                               (CuPtr{Float64}, Int64, CuPtr{Int64}, Int64, Cdouble, Cint, CuPtr{Int64}, CuPtr{Int32},
                                Int64, Ptr{Cvoid}),
                               rec, N, seg, T, x_max, self_loop, offsets, nbr, total[], stream()))
    return _temporal_snapshots(offsets, nbr, n, T, :in, true, kws)   # GNNGraph(adj)'s order, A[nz] = 1 as weights
end

## Link prediction on device COO graphs — replace negative_sample (GNNGraphs/src/transform.jl:890-929: a host copy,
## randsubseq over all n² codes, setdiff!), rand_edge_split (:945-968), perturb_edges (:385-418), intersect
## (operators.jl:7-20) and edge_encoding / edge_decoding (utils.jl:189-268).  One primitive, gnnb_sample_codes: the first
## m codes of a seeded permutation of [0, M) outside a sorted exclusion set, in permutation order.  Codes are the
## reference's idx - 1 (UInt64); randomness comes from `seed` (drawn from `rng` when none is given).
const CuCOO = Tuple{<:CuVector{<:Integer}, <:CuVector{<:Integer}, <:Any}
const SPACE = Dict((true, true) => Cint(0), (true, false) => Cint(1), (false, true) => Cint(2), (false, false) => Cint(3))
_space_size(sp, n) = (n * n, n * (n - 1), n * (n + 1) ÷ 2, n * (n - 1) ÷ 2)[sp + 1]
_seed(rng, seed) = seed === nothing ? rand(rng, UInt64) : UInt64(seed)

function _encode(sp::Cint, n, s::CuVector{Int64}, t::CuVector{Int64})
    codes = CuVector{UInt64}(undef, length(s))
    check(ccall((:gnnb_edge_encode, LIB), Cint,
                (Cint, Int64, Int64, CuPtr{Int64}, CuPtr{Int64}, Int64, Cint, CuPtr{UInt64}, Ptr{Cvoid}),
                sp, n, n, s, t, length(s), 1, codes, stream()))
    codes
end

function _decode(sp::Cint, n1, n2, codes::CuVector{UInt64})
    s, t = CuVector{Int64}(undef, length(codes)), CuVector{Int64}(undef, length(codes))
    check(ccall((:gnnb_edge_decode, LIB), Cint,
                (Cint, Int64, Int64, CuPtr{UInt64}, Int64, Cint, CuPtr{Int64}, CuPtr{Int64}, Ptr{Cvoid}),
                sp, n1, n2, codes, length(codes), 1, s, t, stream()))
    s, t
end

function _codes_sorted(sp::Cint, n, s::CuVector{Int64}, t::CuVector{Int64})
    out = CuVector{UInt64}(undef, length(s))
    cnt = Ref{Int64}(0)
    check(ccall((:gnnb_edge_codes_sorted, LIB), Cint,
                (Cint, Int64, Int64, CuPtr{Int64}, CuPtr{Int64}, Int64, Cint, CuPtr{UInt64}, Ref{Int64}, Ptr{Cvoid}),
                sp, n, n, s, t, length(s), 1, out, cnt, stream()))
    out[1:cnt[]]
end

function _sample_codes(M::Integer, m::Integer, excl::Union{Nothing, CuVector{UInt64}}, seed::UInt64)
    x = excl === nothing ? 0 : length(excl)
    out = CuVector{UInt64}(undef, max(0, min(m, M - x)))
    cnt = Ref{Int64}(0)
    check(ccall((:gnnb_sample_codes, LIB), Cint,
                (UInt64, CuPtr{UInt64}, Int64, Int64, UInt64, CuPtr{UInt64}, Ref{Int64}, Ptr{Cvoid}),
                M, excl === nothing ? CU_NULL : excl, x, m, seed, out, cnt, stream()))
    out[1:cnt[]]
end

function GNNGraphs.edge_encoding(s::CuVector{<:Integer}, t::CuVector{<:Integer}, n; directed = true, self_loops = true)
    sp = SPACE[(directed, self_loops)]
    return _encode(sp, n, CuVector{Int64}(s), CuVector{Int64}(t)) .+ UInt64(1), _space_size(sp, n)
end

function GNNGraphs.edge_decoding(idx::CuVector{<:Integer}, n; directed = true, self_loops = true)
    return _decode(SPACE[(directed, self_loops)], n, n, CuVector{UInt64}(idx) .- UInt64(1))
end

GNNGraphs.edge_decoding(idx::CuVector{<:Integer}, n1, n2) = _decode(Cint(4), n1, n2, CuVector{UInt64}(idx) .- UInt64(1))

function GNNGraphs.negative_sample(g::GNNGraph{<:CuCOO}; max_trials = 3, num_neg_edges = g.num_edges,
                                   bidirected = GNNGraphs.is_bidirected(g), seed = nothing, rng = Random.default_rng())
    @assert g.num_graphs == 1
    n = g.num_nodes
    @assert n >= 2 "negative_sample needs at least 2 nodes"
    s, t = CuVector{Int64}.(edge_index(g))
    sp = bidirected ? Cint(3) : Cint(1)                        # no self loops; undirected pairs when bidirected
    codes = _sample_codes(_space_size(sp, n), bidirected ? num_neg_edges ÷ 2 : num_neg_edges,
                          _codes_sorted(sp, n, s, t), _seed(rng, seed))
    sn, tn = _decode(sp, n, n, codes)
    if bidirected
        sn, tn = vcat(sn, tn), vcat(tn, sn)
    end
    return GNNGraph(sn, tn, num_nodes = n)
end

function GNNGraphs.rand_edge_split(g::GNNGraph{<:CuCOO}, frac; bidirected = GNNGraphs.is_bidirected(g),
                                   seed = nothing, rng = Random.default_rng())
    @assert 0 <= frac <= 1 "frac must be between 0 and 1"
    s, t = edge_index(g)
    if bidirected
        @assert GNNGraphs.is_bidirected(g)
        @assert !GNNGraphs.has_self_loops(g)
        @assert !GNNGraphs.has_multi_edges(g)
        mask = s .< t
        s, t = s[mask], t[mask]
    end
    ne = length(s)
    eids = Int64.(_sample_codes(ne, ne, nothing, _seed(rng, seed))) .+ 1
    size1 = round(Int, ne * frac)
    e1, e2 = eids[1:size1], eids[(size1 + 1):end]
    s1, t1, s2, t2 = s[e1], t[e1], s[e2], t[e2]
    if bidirected
        s1, t1 = vcat(s1, t1), vcat(t1, s1)
        s2, t2 = vcat(s2, t2), vcat(t2, s2)
    end
    return GNNGraph(s1, t1, num_nodes = g.num_nodes), GNNGraph(s2, t2, num_nodes = g.num_nodes)
end

function GNNGraphs.perturb_edges(g::GNNGraph{<:CuCOO}, perturb_ratio::AbstractFloat; seed = nothing,
                                 rng = Random.default_rng())
    @assert perturb_ratio >= 0 && perturb_ratio <= 1 "perturb_ratio must be between 0 and 1"
    k = ceil(Int, g.num_edges * perturb_ratio)
    k == 0 && return g
    n = g.num_nodes
    @assert n > 1 "Graph must contain at least 2 nodes to add edges"
    @assert k <= n * (n - 1)
    snew, tnew = _decode(Cint(1), n, n, _sample_codes(n * (n - 1), k, nothing, _seed(rng, seed)))
    return GNNGraphs.add_edges(g, (snew, tnew, nothing))
end

function Base.intersect(g1::GNNGraph{<:CuCOO}, g2::GNNGraph{<:CuCOO})
    @assert g1.num_nodes == g2.num_nodes
    n = g1.num_nodes
    s1, t1 = CuVector{Int64}.(edge_index(g1))
    s2, t2 = CuVector{Int64}.(edge_index(g2))
    (isempty(s1) || isempty(s2)) && return GNNGraph(s1[1:0], t1[1:0]; num_nodes = n)
    codes1 = _encode(Cint(0), n, s1, t1)
    set2 = _codes_sorted(Cint(0), n, s2, t2)
    inb = CuVector{UInt8}(undef, length(codes1))
    check(ccall((:gnnb_codes_member, LIB), Cint, (CuPtr{UInt64}, Int64, CuPtr{UInt64}, Int64, CuPtr{UInt8}, Ptr{Cvoid}),
                codes1, length(codes1), set2, length(set2), inb, stream()))
    # first occurrence of every pair of g1 (Julia's intersect keeps g1's order, each element once): the run heads of the
    # stable pair sort of gnnb_coalesce_edges
    E = length(s1)
    so, to = similar(s1), similar(t1)
    perm, seg = CuVector{Int64}(undef, E), CuVector{Int64}(undef, E)
    nu = Ref{Int64}(0)
    check(ccall((:gnnb_coalesce_edges, LIB), Cint,
                (CuPtr{Int64}, CuPtr{Int64}, Int64, Int64, Cint, Cint, CuPtr{Int64}, CuPtr{Int64}, CuPtr{Int64},
                 CuPtr{Int64}, Ref{Int64}, Ptr{Cvoid}),
                s1, t1, E, n, 8, 1, so, to, perm, seg, nu, stream()))
    head = vcat(CUDA.ones(Bool, 1), seg[2:end] .!= seg[1:end-1])
    first = CUDA.zeros(Bool, E)
    first[perm[head] .+ 1] .= true
    keep = findall((inb .!= 0) .& first)
    return GNNGraph(s1[keep], t1[keep]; num_nodes = n)
end

## Graph editing on device COO graphs — replace remove_edges (GNNGraphs/src/transform.jl:121-147), remove_nodes
## (:212-276), getgraph (:825-888) and add_nodes (:553-563).  One entry, gnnb_graph_subgraph: kept nodes renumbered in
## ascending old id, kept edges in COO order, and, when the parent has a plan and at most DERIVE_MAX_EDGES edges, the child's
## plan derived from the parent's CSR (no sort) and registered in the plan cache under the child's index arrays; the
## same arrays come from the masks otherwise (the Python mirror's policy).  Drops with probability p are gnnb_bernoulli_keep, keyed by `seed`
## (drawn from `rng` when none is given).  The deliberate differences of the Python mirror hold here too
## (graphneuralnetworks.jl_b200/transform.py): graph_indicator is sliced by remove_nodes and extended by add_nodes, and
## getgraph keeps an edge only when both of its endpoints are kept.
function _drop_mask(k::Integer, p, seed::UInt64)
    keep = CuVector{UInt8}(undef, k)
    check(ccall((:gnnb_bernoulli_keep, LIB), Cint, (Int64, Cdouble, UInt64, CuPtr{UInt8}, Ptr{Cvoid}),
                k, Float64(p), seed, k == 0 ? CU_NULL : keep, stream()))
    keep
end

function _id_mask(ids, k::Integer)
    keep = CUDA.ones(UInt8, k)
    if !isempty(ids)
        @assert 1 <= minimum(ids) && maximum(ids) <= k "id out of range 1:$k"
        keep[CuVector{Int64}(ids)] .= 0x00
    end
    keep
end

# the plan of g if one is cached, without building one
function cached_plan(g::GNNGraph{<:COO_T})
    s, t = edge_index(g)
    lock(PLANS_LOCK) do
        for en in get(PLANS, s, PlanEntry[])
            (en.t.value === t && en.num_nodes == g.num_nodes && en.num_edges == g.num_edges) && return en.plan
        end
        return nothing
    end
end

# Derive the child's plan only when g has one and at most this many edges (the Python mirror's
# transform._DERIVE_MAX_EDGES, measured in DESIGN.md §7); otherwise the child's plan is a fresh sort when first used.
const DERIVE_MAX_EDGES = 1 << 23

# (s, t, num_nodes, kept edge ids (1-based), old ids of the kept nodes (1-based)); a derived plan goes into the cache
function _subgraph(g::GNNGraph{<:CuCOO}, node_keep, edge_keep, extra::Integer)
    n, E = g.num_nodes, g.num_edges
    s, t = edge_index(g)
    p = cached_plan(g)
    if p !== nothing && E <= DERIVE_MAX_EDGES
        nmap = CuVector{Int32}(undef, n)
        kept = CuVector{Int64}(undef, E)
        h, n2, e2 = Ref{Ptr{Cvoid}}(C_NULL), Ref{Int64}(0), Ref{Int64}(0)
        check(ccall((:gnnb_graph_subgraph, LIB), Cint,
                    (Ptr{Cvoid}, CuPtr{UInt8}, CuPtr{UInt8}, Int64, Ref{Ptr{Cvoid}}, CuPtr{Int32}, CuPtr{Int64},
                     Ref{Int64}, Ref{Int64}, Ptr{Cvoid}),
                    p.h, cuptr(node_keep), cuptr(edge_keep), extra, h, n == 0 ? CU_NULL : nmap,
                    E == 0 ? CU_NULL : kept, n2, e2, stream()))
        child, num_nodes = Plan(h[]), Int(n2[])
        kept = kept[1:e2[]] .+ 1
    else
        child = nothing
        ek = edge_keep === nothing ? CUDA.ones(Bool, E) : edge_keep .!= 0x00
        num_nodes = n + extra
        if node_keep !== nothing
            nk = node_keep .!= 0x00
            ek = ek .& nk[s] .& nk[t]
            nmap = Int32.(cumsum(nk)) .- Int32(1)
            num_nodes = Int(sum(nk)) + extra
        end
        @assert num_nodes < 2^31 - 1 "kept nodes + extra nodes = $num_nodes must be < 2^31-1"
        kept = findall(ek)
    end
    s, t = s[kept], t[kept]
    if node_keep !== nothing
        s, t = eltype(s).(nmap[s] .+ 1), eltype(t).(nmap[t] .+ 1)
    end
    if child !== nothing
        lock(PLANS_LOCK) do
            push!(get!(() -> PlanEntry[], PLANS, s), PlanEntry(WeakRef(t), num_nodes, length(s), child))
        end
    end
    nodes = node_keep === nothing ? CuVector{Int64}(1:n) : findall(node_keep .!= 0x00)
    return s, t, num_nodes, kept, nodes
end

_take(x::Nothing, idx) = nothing
_take(x, idx) = GNNGraphs.getobs(x, idx)

function GNNGraphs.remove_edges(g::GNNGraph{<:CuCOO}, edges_to_remove::AbstractVector{<:Integer})
    s, t, n, kept, _ = _subgraph(g, nothing, _id_mask(edges_to_remove, g.num_edges), 0)
    return GNNGraph((s, t, _take(get_edge_weight(g), kept)), n, length(s), g.num_graphs, g.graph_indicator, g.ndata,
                    _take(g.edata, kept), g.gdata)
end

function GNNGraphs.remove_edges(g::GNNGraph{<:CuCOO}, p::AbstractFloat; seed = nothing, rng = Random.default_rng())
    s, t, n, kept, _ = _subgraph(g, nothing, _drop_mask(g.num_edges, p, _seed(rng, seed)), 0)
    return GNNGraph((s, t, _take(get_edge_weight(g), kept)), n, length(s), g.num_graphs, g.graph_indicator, g.ndata,
                    _take(g.edata, kept), g.gdata)
end

function _remove_nodes(g::GNNGraph{<:CuCOO}, keep)
    s, t, n, kept, nodes = _subgraph(g, keep, nothing, 0)
    gi = g.graph_indicator === nothing ? nothing : g.graph_indicator[nodes]
    return GNNGraph((s, t, _take(get_edge_weight(g), kept)), n, length(s), g.num_graphs, gi, _take(g.ndata, nodes),
                    _take(g.edata, kept), g.gdata)
end

GNNGraphs.remove_nodes(g::GNNGraph{<:CuCOO}, nodes_to_remove::AbstractVector{<:Integer}) =
    _remove_nodes(g, _id_mask(nodes_to_remove, g.num_nodes))

GNNGraphs.remove_nodes(g::GNNGraph{<:CuCOO}, p::AbstractFloat; seed = nothing, rng = Random.default_rng()) =
    _remove_nodes(g, _drop_mask(g.num_nodes, p, _seed(rng, seed)))

function GNNGraphs.getgraph(g::GNNGraph{<:CuCOO}, i::AbstractVector{Int}; nmap = false)
    if g.graph_indicator === nothing
        @assert i == [1]
        return nmap ? (g, 1:(g.num_nodes)) : g
    end
    @assert all(1 .<= i .<= g.num_graphs) "graph id out of range 1:$(g.num_graphs)"
    lut = zeros(Int, g.num_graphs)
    for (pos, v) in enumerate(i)                               # the reference's Dict: a repeated id takes its last position
        lut[v] = pos
    end
    gi = CuVector(lut)[g.graph_indicator]
    keep = UInt8.(gi .> 0)
    s, t, n, kept, nodes = _subgraph(g, keep, nothing, 0)
    gnew = GNNGraph((s, t, _take(get_edge_weight(g), kept)), n, length(s), length(i), gi[nodes], _take(g.ndata, nodes),
                    _take(g.edata, kept), _take(g.gdata, i))
    return nmap ? (gnew, nodes) : gnew
end

function GNNGraphs.add_nodes(g::GNNGraph{<:CuCOO}, n::Integer; ndata = (;))
    ndata = GNNGraphs.normalize_graphdata(ndata, default_name = :x, n = n)
    ndata = GNNGraphs.cat_features(g.ndata, ndata)
    s, t, num_nodes, _, _ = _subgraph(g, nothing, nothing, n)
    gi = g.graph_indicator === nothing ? nothing : vcat(g.graph_indicator, fill!(similar(g.graph_indicator, n), g.num_graphs))
    return GNNGraph((s, t, get_edge_weight(g)), num_nodes, length(s), g.num_graphs, gi, ndata, g.edata, g.gdata)
end

## random_walk_pe on device COO graphs — replaces GNNGraphs/src/transform.jl:975-990 (K products of the dense N x N
## matrix RW = A * Diagonal(deg_inv), which for a batch of 10 000 molecules is 212 GB per matrix).  The walks of each graph
## of the batch run in shared memory (gnnb_random_walk_pe); a graph above RWPE_SMEM_MAX_NODES is composed from the fused
## propagate on its derived plan, 128 sources at a time.  Same routing and same bits as the Python mirror
## (graphneuralnetworks.jl_b200/transform.py): segments = runs of a non-decreasing graph_indicator that no edge crosses,
## otherwise the whole graph.
const RWPE_SMEM_MAX_NODES = 896                               # GNNB_RWPE_SMEM_MAX_NODES

function _rwpe_propagate!(out::CuMatrix{Float32}, p::Plan, n::Integer, w, dinv::CuVector{Float32}, K::Integer)
    D = 128
    w = (w === nothing || isempty(w)) ? nothing : w
    x, y = CUDA.zeros(Float32, D, n), CUDA.zeros(Float32, D, n)
    for b0 in 0:D:(n - 1)
        nb = min(D, n - b0)
        lin = CuVector{Int64}((b0 .+ (0:nb-1)) .* D .+ (1:nb))  # x[c, b0 + c] in column-major (D, n)
        fill!(x, 0f0)
        x[lin] .= 1f0
        for k in 1:K
            check(ccall((:gnnb_propagate, LIB), Cint,
                        (Ptr{Cvoid}, Cint, Cint, Cint, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32},
                         Int64, CuPtr{Float32}, Ptr{Cvoid}),
                        p.h, 0, w === nothing ? 0 : 1, 0, x, cuptr(w), CU_NULL, dinv, D, y, stream()))
            out[k, (b0 + 1):(b0 + nb)] .= y[lin]
            x, y = y, x
        end
    end
    return out
end

function GNNGraphs.random_walk_pe(g::GNNGraph{<:CuCOO}, walk_length::Int)
    @assert walk_length >= 1 "walk_length = $walk_length must be >= 1"
    n, K = g.num_nodes, walk_length
    out = CuMatrix{Float32}(undef, K, n)                      # column j = PE[1:K, j]: node-major, as the entry writes it
    n == 0 && return out
    p = plan(g)
    w = get_edge_weight(g)
    w = w === nothing ? nothing : CuVector{Float32}(w)
    deg = CUDA.zeros(Float32, n)
    check(ccall((:gnnb_degree, LIB), Cint, (Ptr{Cvoid}, Cint, CuPtr{Float32}, CuPtr{Float32}, Ptr{Cvoid}),
                p.h, 0, cuptr(w), deg, stream()))
    dinv = inv.(deg)
    dinv[isinf.(dinv)] .= 0f0
    seg = nothing
    if g.graph_indicator !== nothing
        order, _, sg = _knn_segments(g.graph_indicator, n)
        gi = CuVector{Int64}(g.graph_indicator)
        s, t = edge_index(g)
        if order === nothing && sg !== nothing && all(gi[s] .== gi[t])
            seg = sg
        end
    end
    sp, ns = _knn_seg_args(seg)
    sizes = seg === nothing ? [n] : Array(seg[2:end] .- seg[1:end-1])
    big = findall(sizes .> RWPE_SMEM_MAX_NODES)
    if length(big) < ns
        check(ccall((:gnnb_random_walk_pe, LIB), Cint,
                    (Ptr{Cvoid}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Int64}, Int64, Cint, CuPtr{Float32}, Ptr{Cvoid}),
                    p.h, cuptr(w), dinv, sp, ns, K, out, stream()))
    end
    for i in big
        if seg === nothing
            _rwpe_propagate!(out, p, n, w, dinv, K)
            continue
        end
        a, b = Array(seg[i:i+1])
        keep = CUDA.zeros(UInt8, n)
        keep[(a + 1):b] .= 0x01
        s, t, m, kept, _ = _subgraph(g, keep, nothing, 0)
        h = GNNGraph(s, t; num_nodes = m)
        ws = w === nothing ? nothing : w[kept]
        sub = view(out, :, (a + 1):b)
        tmp = CuMatrix{Float32}(undef, K, m)
        _rwpe_propagate!(tmp, plan(h), m, ws, dinv[(a + 1):b], K)
        sub .= tmp
    end
    return out
end
ChainRulesCore.@non_differentiable GNNGraphs.random_walk_pe(::Any...)

## ppr_diffusion on device COO graphs — replaces GNNGraphs/src/transform.jl:1026-1051 (`inv` of the dense N x N matrix
## I + (alpha - 1) A of the whole batch).  The inverse of a block-diagonal matrix is block-diagonal: each graph of the
## batch of at most PPR_SMEM_MAX_NODES nodes is inverted in shared memory (gnnb_ppr_diffusion); a larger one is built by
## gnnb_ppr_matrix into an identity-padded matrix and inverted densely.  Same routing as the Python mirror
## (graphneuralnetworks.jl_b200/transform.py): segments = runs of a non-decreasing graph_indicator that no edge crosses,
## otherwise the whole graph.
const PPR_SMEM_MAX_NODES = 240                                # GNNB_PPR_SMEM_MAX_NODES
const PPR_PAD = 128

function GNNGraphs.ppr_diffusion(g::GNNGraph{<:CuCOO}; alpha = 0.85f0)
    n, E = g.num_nodes, g.num_edges
    s, t = edge_index(g)
    w_out = CuVector{Float32}(undef, E)
    (n == 0 || E == 0) && return GNNGraph((s, t, w_out), n, E, g.num_graphs, g.graph_indicator, g.ndata, g.edata, g.gdata)
    a32 = Float32(alpha)
    p = plan(g)
    w = get_edge_weight(g)
    w = w === nothing ? nothing : CuVector{Float32}(w)
    seg = nothing
    if g.graph_indicator !== nothing
        order, _, sg = _knn_segments(g.graph_indicator, n)
        gi = CuVector{Int64}(g.graph_indicator)
        if order === nothing && sg !== nothing && all(gi[s] .== gi[t])
            seg = sg
        end
    end
    sp, ns = _knn_seg_args(seg)
    bounds = seg === nothing ? [0, n] : Array(seg)
    sizes = bounds[2:end] .- bounds[1:end-1]
    big = findall(sizes .> PPR_SMEM_MAX_NODES)
    if length(big) < ns
        info = CuVector{Int32}(undef, ns)
        check(ccall((:gnnb_ppr_diffusion, LIB), Cint,
                    (Ptr{Cvoid}, CuPtr{Float32}, Cfloat, CuPtr{Int64}, Int64, CuPtr{Float32}, CuPtr{Int32}, Ptr{Cvoid}),
                    p.h, cuptr(w), a32, sp, ns, w_out, info, stream()))
        hinfo = Array(info)
        i = findfirst(>(0), hinfo)
        i === nothing || throw(SingularException(Int(hinfo[i])))   # the zero pivot's step, as LAPACK's info
    end
    for i in big
        a, b = bounds[i], bounds[i + 1]
        m = b - a
        P = cld(m, PPR_PAD) * PPR_PAD
        M = CuMatrix{Float32}(I, P, P)
        # gnnb_ppr_matrix writes row-major rows of M; a column-major P x P buffer holds them as its transpose
        check(ccall((:gnnb_ppr_matrix, LIB), Cint,
                    (Ptr{Cvoid}, CuPtr{Float32}, Cfloat, Int64, Int64, Int64, CuPtr{Float32}, Ptr{Cvoid}),
                    p.h, cuptr(w), a32, a, b, P, M, stream()))
        Minv = inv(M)                                         # SingularException for a singular block
        sel = findall((t .> a) .& (t .<= b))                  # the graph's edges (none crosses it)
        idx = CartesianIndex.(Int.(s[sel]) .- a, Int.(t[sel]) .- a)   # (M^T)^-1 = (M^-1)^T: [s, t] of the transpose
        w_out[sel] .= a32 .* Minv[idx]
    end
    return GNNGraph((s, t, w_out), n, E, g.num_graphs, g.graph_indicator, g.ndata, g.edata, g.gdata)
end
ChainRulesCore.@non_differentiable GNNGraphs.ppr_diffusion(::Any...)

## laplacian_lambda_max on device COO graphs — replaces GNNGraphs/src/query.jl:598-610 (per graph a getgraph, a
## normalized_laplacian and KrylovKit's eigsolve(Symmetric(L), ...) on the host).  A graph, or every graph of a batch,
## of at most LMAX_SMEM_MAX_NODES nodes: gnnb_laplacian_lambda_max, in one call.  Larger ones: the reference's own method
## through getgraph.  The degrees are the reference's row sums of A (dir = :out) or A' (every other dir), plus 1 under
## add_self_loops.
const LMAX_SMEM_MAX_NODES = 169                               # GNNB_LMAX_SMEM_MAX_NODES

function _lmax_entry(g::GNNGraph, seg, ns, add_self_loops::Bool, dir::Symbol)
    w = get_edge_weight(g)
    w = w === nothing ? nothing : CuVector{Float32}(w)
    deg = CuVector{Float32}(degree(g, Float32; dir = dir == :out ? :out : :in))
    add_self_loops && (deg .+= 1f0)
    @assert all(!iszero, Array(deg)) "Graph contains isolated nodes, cannot compute `normalized_adjacency`."
    out = CuVector{Float64}(undef, ns)
    info = CuVector{Int32}(undef, ns)
    sp, _ = _knn_seg_args(seg)
    d = dir == :out ? Cint(0) : (dir == :in ? Cint(1) : Cint(2))
    check(ccall((:gnnb_laplacian_lambda_max, LIB), Cint,
                (Ptr{Cvoid}, CuPtr{Float32}, CuPtr{Float32}, Cint, Cint, CuPtr{Int64}, Int64, CuPtr{Float64},
                 CuPtr{Int32}, Ptr{Cvoid}),
                plan(g).h, cuptr(w), deg, d, Cint(add_self_loops), sp, ns, out, info, stream()))
    return Array(out), Array(info)
end

function GNNGraphs.laplacian_lambda_max(g::GNNGraph{<:CuCOO}, T::DataType = Float32;
                                        add_self_loops::Bool = false, dir::Symbol = :out)
    if g.num_graphs == 1
        g.num_nodes <= LMAX_SMEM_MAX_NODES || return invoke(GNNGraphs.laplacian_lambda_max, Tuple{GNNGraph, DataType},
                                                            g, T; add_self_loops, dir)
        return T(_lmax_entry(g, nothing, 1, add_self_loops, dir)[1][1])
    end
    eigenvalues = zeros(g.num_graphs)
    gi = g.graph_indicator
    order, _, seg = _knn_segments(gi, g.num_nodes)
    s, t = edge_index(g)
    giv = CuVector{Int64}(gi)
    if order === nothing && seg !== nothing && length(seg) == g.num_graphs + 1 && all(giv[s] .== giv[t])
        vals, info = _lmax_entry(g, seg, g.num_graphs, add_self_loops, dir)
        for i in 1:(g.num_graphs)
            eigenvalues[i] = info[i] == 0 ? vals[i] :
                             GNNGraphs._eigmax(normalized_laplacian(getgraph(g, i), T; add_self_loops, dir))
        end
        return eigenvalues
    end
    for i in 1:(g.num_graphs)                                 # getgraph semantics, graph by graph
        eigenvalues[i] = laplacian_lambda_max(getgraph(g, i), T; add_self_loops, dir)
    end
    return eigenvalues
end
ChainRulesCore.@non_differentiable GNNGraphs.laplacian_lambda_max(::Any...)

## color_refinement on device COO graphs — replaces GNNGraphs/src/utils.jl:340-389 (a host loop that hashes
## (x_i, sort(x[in-neighbours])) into a Dict and indexes scalars, so it cannot run on a CuArray graph).  One pass of
## gnnb_color_refinement's signature kernel per round and a stable radix sort of the exact (c_i, S_1, S_2) key.  Same
## contract as the Python mirror (graphneuralnetworks.jl_b200/transform.py): rounds until the class count stops
## changing (the reference stops after at most two; `max_iters = 2` gives its partition), colours 1..k by first
## appearance renumbered every round, signatures grouped by a mod 2^61 - 1 multiset hash.
function GNNGraphs.color_refinement(g::GNNGraph{<:CuCOO}, x0::AbstractVector{<:Integer} = CUDA.ones(Int, g.num_nodes);
                                    max_iters::Union{Nothing,Integer} = nothing)
    @assert length(x0) == g.num_nodes "length(x0) = $(length(x0)) must equal num_nodes = $(g.num_nodes)"
    @assert max_iters === nothing || max_iters >= 1 "max_iters = $max_iters must be nothing or >= 1"
    n = g.num_nodes
    x = CuVector{Int64}(undef, n)
    n == 0 && return x, 0, 1
    p = plan(g)
    xd = CuVector{Int64}(x0)
    k, it = Ref{Int64}(0), Ref{Int64}(0)
    check(ccall((:gnnb_color_refinement, LIB), Cint,
                (Ptr{Cvoid}, CuPtr{Int64}, Int64, CuPtr{Int64}, Ref{Int64}, Ref{Int64}, Ptr{Cvoid}),
                p.h, xd, max_iters === nothing ? 0 : max_iters, x, k, it, stream()))
    return x, Int(k[]), Int(it[])
end
ChainRulesCore.@non_differentiable GNNGraphs.color_refinement(::Any...)

## set2set_pool on device COO graphs — replaces GNNlib/src/layers/pool.jl:29-43.  Each iteration's attention
## (broadcast_nodes, sum(qn .* x), softmax_nodes, reduce_nodes: about six passes over D x N floats and three D x N
## temporaries) is one pass of gnnb_set2set_attend over the graph-indicator plan (node k -> graph indicator[k]); its rrule
## calls gnnb_set2set_attend_bwd, whose per-edge dxe is dx on that plan, and keeps only graph-sized state besides x and q.
## Same routing as the Python mirror (graphneuralnetworks.jl_b200/readout.py): n_in above SET2SET_MAX_D takes the
## reference's composition.
const SET2SET_MAX_D = 1024                                    # GNNB_SET2SET_MAX_D

function _indicator_plan(g::GNNGraph)
    n = g.num_nodes
    gi = g.graph_indicator === nothing ? CUDA.ones(Int64, n) : CuVector{Int64}(g.graph_indicator)
    src = CuVector{Int64}(1:n)
    h = Ref{Ptr{Cvoid}}(C_NULL)
    check(ccall((:gnnb_graph_create, LIB), Cint,
                (Ref{Ptr{Cvoid}}, CuPtr{Cvoid}, CuPtr{Cvoid}, Int64, Int64, Int64, Cint, Cint, Cint, Ptr{Cvoid}),
                h, pointer(src), pointer(gi), n, n, g.num_graphs, 8, 1, 1, stream()))
    return Plan(h[])
end
ChainRulesCore.@non_differentiable _indicator_plan(::Any...)

function _set2set_attend(p::Plan, x::CuMatrix{Float32}, q::CuMatrix{Float32})
    D, G = size(q)
    r = similar(q)
    smax, ssum = CuVector{Float32}(undef, G), CuVector{Float32}(undef, G)
    check(ccall((:gnnb_set2set_attend, LIB), Cint,
                (Ptr{Cvoid}, CuPtr{Float32}, CuPtr{Float32}, Int64, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32},
                 Ptr{Cvoid}),
                p.h, x, q, D, r, smax, ssum, stream()))
    return r, smax, ssum
end

set2set_attend(p::Plan, x::CuMatrix{Float32}, q::CuMatrix{Float32}) = _set2set_attend(p, x, q)[1]

function ChainRulesCore.rrule(::typeof(set2set_attend), p::Plan, x::CuMatrix{Float32}, q::CuMatrix{Float32})
    r, smax, ssum = _set2set_attend(p, x, q)
    function set2set_attend_pullback(Δ)
        dr = CuMatrix{Float32}(unthunk(Δ))
        dx, dq = similar(x), similar(q)
        check(ccall((:gnnb_set2set_attend_bwd, LIB), Cint,
                    (Ptr{Cvoid}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32},
                     CuPtr{Float32}, Int64, CuPtr{Float32}, CuPtr{Float32}, Ptr{Cvoid}),
                    p.h, x, q, r, smax, ssum, dr, size(q, 1), dx, dq, stream()))
        return NoTangent(), NoTangent(), dx, dq
    end
    return r, set2set_attend_pullback
end

function GNNlib.set2set_pool(l, g::GNNGraph{<:CuCOO}, x::CuMatrix{Float32})
    @assert size(x, 2) == g.num_nodes "x has $(size(x, 2)) columns instead of num_nodes = $(g.num_nodes)"
    n_in = size(x, 1)
    n_in > SET2SET_MAX_D && return invoke(GNNlib.set2set_pool, Tuple{Any, GNNGraph, AbstractMatrix}, l, g, x)
    p = _indicator_plan(g)
    qstar = CUDA.zeros(Float32, 2 * n_in, g.num_graphs)
    h = CUDA.zeros(Float32, size(l.lstm.Wh, 2))
    state = (h, zero(h))
    for _ in 1:l.num_iters
        q, state = l.lstm(qstar, state)
        r = set2set_attend(p, x, CuMatrix{Float32}(q))
        qstar = vcat(q, r)
    end
    return qstar
end

## global_attention_pool on device COO graphs — replaces GNNlib/src/layers/pool.jl:7-12 for a gate of one row:
## softmax_nodes, the D x N product α .* ffeat(x) and reduce_nodes(+) are one pass of gnnb_attention_pool over the
## graph-indicator plan; its rrule calls gnnb_attention_pool_bwd, whose per-edge dfe and dgate_e are df and dgate on that
## plan, and keeps only graph-sized state besides f and the gate.  Other shapes (a gate per channel, D above
## SET2SET_MAX_D) take the reference's composition, as in the Python mirror.
function _attention_pool(p::Plan, f::CuMatrix{Float32}, gate::CuVector{Float32}, G::Integer)
    D = size(f, 1)
    u = CuMatrix{Float32}(undef, D, G)
    smax, ssum = CuVector{Float32}(undef, G), CuVector{Float32}(undef, G)
    check(ccall((:gnnb_attention_pool, LIB), Cint,
                (Ptr{Cvoid}, CuPtr{Float32}, CuPtr{Float32}, Int64, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32},
                 Ptr{Cvoid}),
                p.h, f, gate, D, u, smax, ssum, stream()))
    return u, smax, ssum
end

attention_pool(p::Plan, f::CuMatrix{Float32}, gate::CuVector{Float32}, G::Integer) = _attention_pool(p, f, gate, G)[1]

function ChainRulesCore.rrule(::typeof(attention_pool), p::Plan, f::CuMatrix{Float32}, gate::CuVector{Float32},
                              G::Integer)
    u, smax, ssum = _attention_pool(p, f, gate, G)
    function attention_pool_pullback(Δ)
        du = CuMatrix{Float32}(unthunk(Δ))
        df, dgate = similar(f), similar(gate)
        check(ccall((:gnnb_attention_pool_bwd, LIB), Cint,
                    (Ptr{Cvoid}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32},
                     CuPtr{Float32}, Int64, CuPtr{Float32}, CuPtr{Float32}, Ptr{Cvoid}),
                    p.h, f, gate, u, smax, ssum, du, size(f, 1), df, dgate, stream()))
        return NoTangent(), NoTangent(), df, dgate, NoTangent()
    end
    return u, attention_pool_pullback
end

function GNNlib.global_attention_pool(l, g::GNNGraph{<:CuCOO}, x::AbstractMatrix)
    gate, feats = l.fgate(x), l.ffeat(x)
    if !(gate isa CuMatrix{Float32} && size(gate, 1) == 1 && feats isa CuMatrix{Float32} &&
         1 <= size(feats, 1) <= SET2SET_MAX_D)
        return invoke(GNNlib.global_attention_pool, Tuple{Any, GNNGraph, AbstractArray}, l, g, x)
    end
    @assert size(gate, 2) == size(feats, 2) == g.num_nodes "fgate(x) and ffeat(x) need num_nodes = $(g.num_nodes) columns"
    return attention_pool(_indicator_plan(g), feats, vec(gate), g.num_graphs)
end

## topk_index / topk_pool on device arrays — replace GNNlib/src/layers/pool.jl:14-27.  The selection is gnnb_topk_keep
## (one segment; NaN never kept nor counted, this library's rule), the score and gate are one pass each over X, and the
## rrule of the gate calls gnnb_topk_gate_bwd, which gives dX through the gather and through y, and dp through y.
const KEY_F32, KEY_F64, KEY_I32, KEY_I64 = Cint(0), Cint(1), Cint(2), Cint(3)
_key_type(::Type{Float32}) = KEY_F32
_key_type(::Type{Float64}) = KEY_F64
_key_type(::Type{Int32}) = KEY_I32
_key_type(::Type{Int64}) = KEY_I64

function _topk_keep(y::CuVector{T}, k::Integer) where {T<:Union{Float32, Float64, Int32, Int64}}
    k >= 1 || throw(ArgumentError("topk_index needs k >= 1 (got $k)"))
    n = length(y)
    keep = CuVector{UInt8}(undef, n)
    check(ccall((:gnnb_topk_keep, LIB), Cint,
                (CuPtr{Cvoid}, Cint, Int64, Ptr{Cvoid}, Int64, Int64, Cdouble, CuPtr{UInt8}, Ptr{Cvoid}, Ptr{Cvoid}),
                y, _key_type(T), n, C_NULL, 1, k, 0.0, keep, C_NULL, stream()))
    return keep
end
ChainRulesCore.@non_differentiable _topk_keep(::Any...)

GNNlib.topk_index(y::CuVector{T}, k::Int) where {T<:Union{Float32, Float64, Int32, Int64}} =
    findall(!iszero, _topk_keep(y, k))

function _topk_score(X::CuMatrix{Float32}, p::CuVector{Float32})
    D, n = size(X)
    y = CuVector{Float32}(undef, n)
    check(ccall((:gnnb_topk_score, LIB), Cint, (CuPtr{Float32}, Int64, Int64, CuPtr{Float32}, CuPtr{Float32}, Ptr{Cvoid}),
                X, n, D, p, y, stream()))
    return y
end
ChainRulesCore.@non_differentiable _topk_score(::Any...)

function topk_gate(X::CuMatrix{Float32}, p::CuVector{Float32}, y::CuVector{Float32}, idx::CuVector{Int64})
    D, n = size(X)
    m = length(idx)
    out = CuMatrix{Float32}(undef, D, m)
    check(ccall((:gnnb_topk_gate, LIB), Cint,
                (CuPtr{Float32}, Int64, Int64, CuPtr{Float32}, CuPtr{Int64}, Int64, CuPtr{Float32}, Ptr{Cvoid}, Ptr{Cvoid}),
                X, n, D, y, idx, m, out, C_NULL, stream()))
    return out
end

function ChainRulesCore.rrule(::typeof(topk_gate), X::CuMatrix{Float32}, p::CuVector{Float32}, y::CuVector{Float32},
                              idx::CuVector{Int64})
    out = topk_gate(X, p, y, idx)
    function topk_gate_pullback(Δ)
        dout = CuMatrix{Float32}(unthunk(Δ))
        D, n = size(X)
        dX, dp = similar(X), similar(p)
        check(ccall((:gnnb_topk_gate_bwd, LIB), Cint,
                    (CuPtr{Float32}, Int64, Int64, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Int64}, Int64, CuPtr{Float32},
                     CuPtr{Float32}, CuPtr{Float32}, Ptr{Cvoid}, Ptr{Cvoid}),
                    X, n, D, y, p, idx, length(idx), dout, dX, dp, C_NULL, stream()))
        return NoTangent(), dX, dp, NoTangent(), NoTangent()
    end
    return out, topk_gate_pullback
end

function GNNlib.topk_pool(t, X::CuMatrix{Float32})
    p = CuVector{Float32}(t.p)
    y = _topk_score(X, p)
    idx = ChainRulesCore.ignore_derivatives(() -> CuVector{Int64}(findall(!iszero, _topk_keep(y, t.k)) .- 1))
    ChainRulesCore.ignore_derivatives(() -> (t.Ã .= view(t.A, Array(idx) .+ 1, Array(idx) .+ 1)))
    return topk_gate(X, p, y, idx)
end

## The gates of the recurrent temporal cells (GraphNeuralNetworks/src/layers/temporalconv.jl) — one pass over node
## columns per call instead of the cells' broadcasts.  px (G·D, N): the x-side pre-activations of the G gates ([r; z; n]
## for the GRU cells, [i; f; c; o] for the LSTM); ah the h-side ones; every array a dense CuMatrix (node stride = rows).
## Wiring GConvGRUCell / DCGRUCell / TGCNCell / GConvLSTMCell to these is left to the cells.
function gru_rz(px::CuMatrix{Float32}, ah::CuMatrix{Float32}, h::CuMatrix{Float32})
    D, N = size(h)
    r, z, rh = similar(h), similar(h), similar(h)
    check(ccall((:gnnb_gru_rz, LIB), Cint,
                (CuPtr{Float32}, Int64, CuPtr{Float32}, CuPtr{Float32}, Int64, Int64, CuPtr{Float32}, CuPtr{Float32},
                 CuPtr{Float32}, Ptr{Cvoid}),
                px, size(px, 1), ah, h, N, D, r, z, rh, stream()))
    return r, z, rh
end

function ChainRulesCore.rrule(::typeof(gru_rz), px::CuMatrix{Float32}, ah::CuMatrix{Float32}, h::CuMatrix{Float32})
    r, z, rh = gru_rz(px, ah, h)
    function gru_rz_pullback(Δ)
        D, N = size(h)
        drh, dz = CuMatrix{Float32}(unthunk(Δ[3])), CuMatrix{Float32}(unthunk(Δ[2]))
        dpre, dh = CuMatrix{Float32}(undef, 2D, N), CUDA.zeros(Float32, D, N)
        check(ccall((:gnnb_gru_rz_bwd, LIB), Cint,
                    (CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, Int64, Int64,
                     CuPtr{Float32}, Int64, CuPtr{Float32}, Ptr{Cvoid}),
                    drh, dz, h, r, z, N, D, dpre, 2D, dh, stream()))
        return NoTangent(), vcat(dpre, CUDA.zeros(Float32, size(px, 1) - 2D, N)), dpre, dh
    end
    return (r, z, rh), gru_rz_pullback
end

function gru_out(px::CuMatrix{Float32}, ah_n::CuMatrix{Float32}, h::CuMatrix{Float32}, z::CuMatrix{Float32}, blend::Int)
    D, N = size(h)
    n, hn = similar(h), similar(h)
    check(ccall((:gnnb_gru_out, LIB), Cint,
                (CuPtr{Float32}, Int64, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, Int64, Int64, Cint,
                 CuPtr{Float32}, CuPtr{Float32}, Ptr{Cvoid}),
                px, size(px, 1), ah_n, h, z, N, D, blend, n, hn, stream()))
    return hn, n
end

function ChainRulesCore.rrule(::typeof(gru_out), px::CuMatrix{Float32}, ah_n::CuMatrix{Float32}, h::CuMatrix{Float32},
                              z::CuMatrix{Float32}, blend::Int)
    hn, n = gru_out(px, ah_n, h, z, blend)
    function gru_out_pullback(Δ)
        D, N = size(h)
        dhn = CuMatrix{Float32}(unthunk(Δ[1]))
        dpre, dz, dh = similar(h), similar(h), similar(h)
        check(ccall((:gnnb_gru_out_bwd, LIB), Cint,
                    (CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, Int64, Int64, Cint, CuPtr{Float32},
                     Int64, CuPtr{Float32}, CuPtr{Float32}, Ptr{Cvoid}),
                    dhn, h, z, n, N, D, blend, dpre, D, dz, dh, stream()))
        return NoTangent(), vcat(CUDA.zeros(Float32, 2D, N), dpre), dpre, dh, dz, NoTangent()
    end
    return (hn, n), gru_out_pullback
end

## w: the peepholes vcat(w_i, w_f, w_c, w_o) (4D), or nothing for Flux's LSTMCell
function _lstm_cell(px, ah, c::CuMatrix{Float32}, w)
    D, N = size(c)
    gates, cn, hn = CuMatrix{Float32}(undef, 4D, N), similar(c), similar(c)
    check(ccall((:gnnb_lstm_cell, LIB), Cint,
                (CuPtr{Float32}, Int64, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, Int64, Int64, CuPtr{Float32},
                 CuPtr{Float32}, CuPtr{Float32}, Ptr{Cvoid}),
                px, size(px, 1), ah, c, w === nothing ? CU_NULL : w, N, D, gates, cn, hn, stream()))
    return hn, cn, gates
end

lstm_cell(px::CuMatrix{Float32}, ah::CuMatrix{Float32}, c::CuMatrix{Float32}, w) = _lstm_cell(px, ah, c, w)[1:2]

function ChainRulesCore.rrule(::typeof(lstm_cell), px::CuMatrix{Float32}, ah::CuMatrix{Float32}, c::CuMatrix{Float32}, w)
    hn, cn, gates = _lstm_cell(px, ah, c, w)
    function lstm_cell_pullback(Δ)
        D, N = size(c)
        dhn = Δ[1] isa AbstractZero ? CUDA.zeros(Float32, D, N) : CuMatrix{Float32}(unthunk(Δ[1]))
        dcn = Δ[2] isa AbstractZero ? CUDA.zeros(Float32, D, N) : CuMatrix{Float32}(unthunk(Δ[2]))
        dpre, dc = CuMatrix{Float32}(undef, 4D, N), similar(c)
        dw = w === nothing ? nothing : similar(w)
        slots = N < 65536 ? cld(N, 64) : 1024                  # GNNB_LSTM_DW_SLOTS(N)
        ws = w === nothing ? nothing : CuVector{Float32}(undef, slots * 4D)
        check(ccall((:gnnb_lstm_cell_bwd, LIB), Cint,
                    (CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, Int64,
                     Int64, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, CuPtr{Float32}, Ptr{Cvoid}),
                    dhn, dcn, c, gates, cn, w === nothing ? CU_NULL : w, N, D, dpre, dc,
                    dw === nothing ? CU_NULL : dw, ws === nothing ? CU_NULL : ws, stream()))
        return NoTangent(), dpre, dpre, dc, w === nothing ? NoTangent() : dw
    end
    return (hn, cn), lstm_cell_pullback
end

end # module
