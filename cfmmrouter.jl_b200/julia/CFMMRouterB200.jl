# CFMMRouterB200.jl -- thin `ccall` shim that keeps CFMMRouter.jl's
# Router / route! / CFMM / Objective API and sends the dual-decomposition inner
# loop (find_arb! sweep + Ψ/acc folds) to libcfmm_b200.so (include/cfmm_b200.h).
#
# STATUS: Julia is not installed in the build image, so this file has never been
# executed; it is written against the C ABI that the Python host
# (cfmmrouter.jl_b200/router.py, same call sequence) exercises in tests/.  It is
# kept deliberately small: everything that is not a ccall is the reference's own
# logic, re-used from the CFMMRouter package (objectives, pool structs, L-BFGS-B).
#
# Usage (drop-in for `using CFMMRouter` on the route! path):
#     using CFMMRouterB200           # re-exports CFMMRouter's names
#     r = B200Router(LinearNonnegative(c), pools, n)    # instead of Router(...)
#     route!(r); netflows(r); r.Δs; r.Λs; r.v           # unchanged
#     route!(r; optimizer=:device)                       # outer iteration on the GPU too (cfmm_solve)
#     r = B200Router(obj, pools, n; devices=0:7)         # pools sharded over 8 GPUs of this process
module CFMMRouterB200

using CFMMRouter
using CFMMRouter: CFMM, ProductTwoCoin, GeometricMeanTwoCoin, UniV3, Objective,
                  f, grad!, lower_limit, upper_limit
using LBFGSB
import CFMMRouter: route!, find_arb!, netflows!, netflows, update_reserves!

export B200Router, sync_reserves!

const LIB = get(ENV, "CFMM_B200_LIB", joinpath(@__DIR__, "..", "libcfmm_b200.so"))

struct B200Error <: Exception
    code::Cint
    msg::String
end

function chk(ctx::Ptr{Cvoid}, rc::Cint)
    rc == 0 && return nothing
    msg = unsafe_string(ccall((:cfmm_last_error, LIB), Cstring, (Ptr{Cvoid},), ctx))
    rc == -1 ? throw(ArgumentError(msg)) : throw(B200Error(rc, msg))   # ArgumentError as the ctors do (cfmms.jl:77-78)
end

# Same fields as Router (src/router.jl:4-10) + the device context and the cached
# folds of the last sweep.
mutable struct B200Router{O,T}
    objective::O
    cfmms::Vector{CFMM{T}}
    Δs::Vector{AbstractVector{T}}
    Λs::Vector{AbstractVector{T}}
    v::Vector{T}
    ctx::Ptr{Cvoid}         # context of the first device (all of them when there is one)
    order::Vector{Int}      # library insertion order -> index into cfmms (first device's shard first)
    ψ::Vector{T}            # Σ A_i(Λ_i − Δ_i) of the last sweep: a view of PINNED memory (cfmm_host_alloc)
    acc::Base.RefValue{T}   # Σ ν[A_i]ᵀ(Λ_i − Δ_i) of the last sweep
    ctxs::Vector{Ptr{Cvoid}}        # one context per device (multi-GPU: pools sharded in list order)
    shard::Vector{UnitRange{Int}}   # positions of `order` each context holds
    pin::Ptr{Float64}               # pinned staging: ν [n] | ψ [n] | acc [1], per context (n_ctx blocks)
    vmat::Vector{T}                 # ν of the last materialising sweep (update_reserves! moves UniV3 pools by it)
end

# One device context holding the pools cfmms[ids] (positions in the caller's list); returns
# (ctx, order) with order = library insertion order -> position in the caller's list.
function make_context(cfmms::Vector{C}, ids::AbstractVector{Int}, n_tokens, device::Integer) where {T,C<:CFMM{T}}
    out = Ref{Ptr{Cvoid}}(C_NULL)
    rc = ccall((:cfmm_create, LIB), Cint, (Ref{Ptr{Cvoid}}, Cint, Int64), out, device, n_tokens)
    rc == 0 || throw(B200Error(rc, unsafe_string(ccall((:cfmm_last_error, LIB), Cstring, (Ptr{Cvoid},), C_NULL))))
    ctx = out[]
    order = Int[]
    prod = [i for i in ids if cfmms[i] isa ProductTwoCoin]
    geo = [i for i in ids if cfmms[i] isa GeometricMeanTwoCoin]
    uni = [i for i in ids if cfmms[i] isa UniV3]
    length(prod) + length(geo) + length(uni) == length(ids) ||
        throw(MethodError(find_arb!, (cfmms,)))    # what the reference would hit
    if !isempty(prod)
        R = Float64[c.R[j] for c in cfmms[prod] for j in 1:2]
        γ = Float64[c.γ for c in cfmms[prod]]
        Ai = Int64[c.Ai[j] for c in cfmms[prod] for j in 1:2]
        GC.@preserve R γ Ai chk(ctx, ccall((:cfmm_add_product, LIB), Cint,
            (Ptr{Cvoid}, Int64, Ptr{Float64}, Ptr{Float64}, Ptr{Int64}), ctx, length(prod), R, γ, Ai))
        append!(order, prod)
    end
    if !isempty(geo)
        R = Float64[c.R[j] for c in cfmms[geo] for j in 1:2]
        w = Float64[c.w[j] for c in cfmms[geo] for j in 1:2]
        γ = Float64[c.γ for c in cfmms[geo]]
        Ai = Int64[c.Ai[j] for c in cfmms[geo] for j in 1:2]
        GC.@preserve R w γ Ai chk(ctx, ccall((:cfmm_add_geomean, LIB), Cint,
            (Ptr{Cvoid}, Int64, Ptr{Float64}, Ptr{Float64}, Ptr{Int64}, Ptr{Float64}), ctx, length(geo), R, γ, Ai, w))
        append!(order, geo)
    end
    if !isempty(uni)
        cp = Float64[c.current_price for c in cfmms[uni]]
        γ = Float64[c.γ for c in cfmms[uni]]
        Ai = Int64[c.Ai[j] for c in cfmms[uni] for j in 1:2]
        off = Int64[0; cumsum(Int64[length(c.lower_ticks) for c in cfmms[uni]])]
        lt = reduce(vcat, (Float64.(c.lower_ticks) for c in cfmms[uni]))
        lq = reduce(vcat, (Float64.(c.liquidity) for c in cfmms[uni]))
        GC.@preserve cp γ Ai off lt lq chk(ctx, ccall((:cfmm_add_univ3, LIB), Cint,
            (Ptr{Cvoid}, Int64, Ptr{Float64}, Ptr{Float64}, Ptr{Int64}, Ptr{Int64}, Ptr{Float64}, Ptr{Float64}),
            ctx, length(uni), cp, γ, Ai, off, lt, lq))
        append!(order, uni)
    end
    chk(ctx, ccall((:cfmm_finalize, LIB), Cint, (Ptr{Cvoid},), ctx))
    return ctx, order
end

# Router(objective, cfmms, n_tokens), src/router.jl:18-35: pack Vector{CFMM} -> SoA, upload.
# devices: one GPU (default) or several of THIS process; the pool list is split into contiguous
# shards, one context per device, and the contexts are joined through the NVLink peer exchange
# (cfmm_comm_export / cfmm_comm_attach, same-process path: raw pointers + peer access), so
# every context's sweep returns the global [ψ; acc].
function B200Router(objective::O, cfmms::Vector{C}, n_tokens; device::Integer=0,
                    devices::AbstractVector{<:Integer}=[device]) where {T,O<:Objective,C<:CFMM{T}}
    T === Float64 || throw(ArgumentError("libcfmm_b200 is fp64-only"))
    W = length(devices)
    m = length(cfmms)
    ctxs = Ptr{Cvoid}[]; order = Int[]; shard = UnitRange{Int}[]
    for (k, dev) in enumerate(devices)
        ids = (div(m * (k - 1), W) + 1):div(m * k, W)
        ctx, ord = make_context(cfmms, collect(ids), n_tokens, dev)
        push!(ctxs, ctx); push!(shard, (length(order) + 1):(length(order) + length(ord))); append!(order, ord)
    end
    if W > 1
        handles = zeros(UInt8, 128 * W)                       # CFMM_COMM_HANDLE_BYTES per context
        for k in 1:W
            GC.@preserve handles chk(ctxs[k], ccall((:cfmm_comm_export, LIB), Cint, (Ptr{Cvoid}, Ptr{UInt8}),
                ctxs[k], pointer(handles, 128 * (k - 1) + 1)))
        end
        for k in 1:W
            GC.@preserve handles chk(ctxs[k], ccall((:cfmm_comm_attach, LIB), Cint,
                (Ptr{Cvoid}, Cint, Cint, Ptr{UInt8}), ctxs[k], W, k - 1, handles))
        end
    end
    # pinned staging per context: the library replays {H2D ν, sweep, D2H [ψ; acc]} as one CUDA
    # graph on buffers it has seen twice (cfmm_b200.h, "sweep_graphs"); pageable Vectors cannot
    pin = convert(Ptr{Float64}, ccall((:cfmm_host_alloc, LIB), Ptr{Cvoid}, (Csize_t,), 8 * (2n_tokens + 1) * W))
    pin == C_NULL && throw(OutOfMemoryError())
    ψ = unsafe_wrap(Array, pin + 8n_tokens, n_tokens)         # context 1's ψ block
    Δs = AbstractVector{T}[zeros(T, 2) for _ in cfmms]     # zerotrade, router.jl:23-26
    Λs = AbstractVector{T}[zeros(T, 2) for _ in cfmms]
    r = B200Router{O,T}(objective, convert(Vector{CFMM{T}}, cfmms), Δs, Λs, zeros(T, n_tokens),
                        ctxs[1], order, ψ, Ref(zero(T)), ctxs, shard, pin, zeros(T, n_tokens))
    finalizer(r) do x
        foreach(c -> ccall((:cfmm_destroy, LIB), Cvoid, (Ptr{Cvoid},), c), x.ctxs)
        ccall((:cfmm_host_free, LIB), Cvoid, (Ptr{Cvoid},), x.pin)
    end
    return r
end

# One dual-gradient sweep on the GPU: find_arb!(r, v) (router.jl:38-42) + both
# folds (router.jl:79-83, 98-100).  materialize=true also refreshes r.Δs / r.Λs.
function sweep!(r::B200Router{O,T}, v::AbstractVector{T}; materialize::Bool=false) where {O,T}
    n = length(r.v); W = length(r.ctxs); blk = 2n + 1
    # ν into every context's pinned block, then one blocking cfmm_sweep per context.  With
    # several contexts the calls MUST run concurrently (the fused exchange kernels wait for
    # each other): one task per context on Julia's thread pool (start julia with -t >= W).
    for k in 1:W
        unsafe_copyto!(r.pin + 8blk * (k - 1), pointer(v), n)
    end
    rcs = zeros(Cint, W)
    GC.@preserve v begin
        @sync for k in 1:W
            base = r.pin + 8blk * (k - 1)
            Threads.@spawn rcs[k] = ccall((:cfmm_sweep, LIB), Cint,
                (Ptr{Cvoid}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Cint),
                r.ctxs[k], base, base + 8n, base + 16n, materialize ? 1 : 0)
        end
    end
    foreach(k -> chk(r.ctxs[k], rcs[k]), 1:W)
    r.acc[] = unsafe_load(r.pin, 2n + 1)            # every context holds the bitwise-identical sum
    if materialize
        r.vmat .= v
        for k in 1:W
            mk = length(r.shard[k])
            D = Vector{Float64}(undef, 2mk); L = Vector{Float64}(undef, 2mk)
            chk(r.ctxs[k], ccall((:cfmm_get_trades, LIB), Cint, (Ptr{Cvoid}, Ptr{Float64}, Ptr{Float64}), r.ctxs[k], D, L))
            for (j, i) in enumerate(r.order[r.shard[k]])   # library order -> r.cfmms order
                r.Δs[i][1] = D[2j-1]; r.Δs[i][2] = D[2j]
                r.Λs[i][1] = L[2j-1]; r.Λs[i][2] = L[2j]
            end
        end
    end
    return nothing
end

find_arb!(r::B200Router, v) = sweep!(r, collect(Float64, v); materialize=true)

# route!, src/router.jl:58-108, with the three find_arb!(r, v) call sites and the
# two fold loops replaced by sweep!.  Everything else is the reference's code path.
# cfmm_solve_opts / cfmm_solve_info of include/cfmm_b200.h
struct SolveOpts; max_iter::Cint; max_fun::Cint; pgtol::Cdouble; factr::Cdouble; end
mutable struct SolveInfo; iterations::Cint; fun_evals::Cint; status::Cint; f::Cdouble; pg_norm::Cdouble; solve_ms::Cdouble; end

# f(ν) = linᵀν on the box for both objectives of the reference (src/objectives.jl:62-79, 106-129)
linear_term(o::CFMMRouter.LinearNonnegative) = zero(o.c)
linear_term(o::CFMMRouter.BasketLiquidation) = (l = copy(o.Δin); l[o.i] = 0; l)

function route!(r::B200Router; v=nothing, verbose=false, m=5, factr=1e1, pgtol=1e-5, maxfun=15_000, maxiter=15_000,
                optimizer::Symbol=:host)
    if optimizer === :device       # the whole outer iteration on the GPU: only scalars cross PCIe
        length(r.ctxs) == 1 || throw(ArgumentError("optimizer=:device drives one GPU"))
        lin = linear_term(r.objective); lo = lower_limit(r.objective); up = upper_limit(r.objective)
        v0 = isnothing(v) ? C_NULL : pointer(v)
        info = SolveInfo(0, 0, 0, 0.0, 0.0, 0.0); opts = SolveOpts(maxiter, maxfun, pgtol, factr)
        GC.@preserve lin lo up v chk(r.ctx, ccall((:cfmm_solve, LIB), Cint,
            (Ptr{Cvoid}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ref{SolveOpts}, Ptr{Float64}, Ref{SolveInfo}),
            r.ctx, lin, lo, up, v0, opts, r.v, info))
        r.vmat .= r.v
        mk = length(r.order); D = Vector{Float64}(undef, 2mk); L = Vector{Float64}(undef, 2mk)
        chk(r.ctx, ccall((:cfmm_get_trades, LIB), Cint, (Ptr{Cvoid}, Ptr{Float64}, Ptr{Float64}), r.ctx, D, L))
        for (j, i) in enumerate(r.order)
            r.Δs[i] .= (D[2j-1], D[2j]); r.Λs[i] .= (L[2j-1], L[2j])
        end
        return nothing
    end
    optimizer = L_BFGS_B(length(r.v), 17)
    if isnothing(v)
        r.v .= ones(length(r.v)) / length(r.v)
    else
        r.v .= v
    end
    bounds = zeros(3, length(r.v))
    bounds[1, :] .= 2
    bounds[2, :] .= lower_limit(r.objective)
    bounds[3, :] .= upper_limit(r.objective)

    function fn(x)                       # router.jl:73-86
        if !all(x .== r.v)
            sweep!(r, x)
            r.v .= x
        end
        return f(r.objective, x) + r.acc[]
    end
    function g!(G, x)                    # router.jl:89-102
        G .= 0
        if !all(x .== r.v)
            sweep!(r, x)
            r.v .= x
        end
        grad!(G, r.objective, x)
        G .+= r.ψ
    end

    sweep!(r, r.v)                       # router.jl:104
    _, x = optimizer(fn, g!, r.v, bounds, m=m, factr=factr, pgtol=pgtol,
                     iprint=verbose ? 1 : -1, maxfun=maxfun, maxiter=maxiter)
    r.v .= x
    sweep!(r, r.v; materialize=true)     # router.jl:107
    return nothing
end

# netflows!, src/router.jl:111-119: host-side pool-order sum of the stored trades
function netflows!(ψ, r::B200Router)
    fill!(ψ, 0)
    for (Δ, Λ, c) in zip(r.Δs, r.Λs, r.cfmms)
        ψ[c.Ai] += Λ - Δ
    end
    return nothing
end
netflows(r::B200Router) = (ψ = zero(r.v); netflows!(ψ, r); ψ)

# The price a UniV3 pool moves to when it trades at ν (cfmm_b200.h, cfmm_apply_trades): the
# same IEEE operations as the device, so the host objects follow the device bit for bit.
function univ3_moved_price(c::UniV3, v)
    q, g = c.current_price, c.γ
    p = v[c.Ai[1]] / v[c.Ai[2]]
    lo = g * q
    (lo <= p && p <= q / g) && return q             # no trade, src/cfmms.jl:347
    target = p < lo ? p / g : g * p                 # upper walk :361 / lower walk :381 (pool price γ·p)
    target > 0 || return q                          # NaN or not > 0: unchanged
    t1 = c.lower_ticks[1]
    return target < t1 ? target : t1
end

# A working update_reserves!(r) (the reference's, src/router.jl:127-132, calls a per-CFMM
# method that is defined nowhere), applied on the device from the materialised trades and
# mirrored on the host objects with the same expressions: R <- R + γΔ − Λ (test/cfmms.jl:10)
# for the two-coin pools; a UniV3 pool moves to the price its walk traded it to.
function update_reserves!(r::B200Router)
    for (Δ, Λ, c) in zip(r.Δs, r.Λs, r.cfmms)
        if c isa ProductTwoCoin || c isa GeometricMeanTwoCoin
            c.R .= c.R .+ c.γ .* Δ .- Λ
        elseif c isa UniV3
            c.current_price = univ3_moved_price(c, r.vmat)
            c.current_tick = searchsortedlast(c.lower_ticks, c.current_price, rev=true)   # cfmms.jl:235
        end
    end
    foreach(c -> chk(c, ccall((:cfmm_apply_trades, LIB), Cint, (Ptr{Cvoid},), c)), r.ctxs)
    return nothing
end

# The reference reads the pool objects live on every sweep; push mutated state explicitly:
# cfmm.R of the two-coin pools, current_price and liquidity of the UniV3 pools (their tick
# prices are fixed at construction).
function sync_reserves!(r::B200Router)
    for (k, ctx) in enumerate(r.ctxs)
        for (ptype, T) in ((0, ProductTwoCoin), (1, GeometricMeanTwoCoin))
            ids = [i for i in r.order[r.shard[k]] if r.cfmms[i] isa T]
            isempty(ids) && continue
            R = Float64[r.cfmms[i].R[j] for i in ids for j in 1:2]
            chk(ctx, ccall((:cfmm_update_reserves, LIB), Cint,
                (Ptr{Cvoid}, Cint, Int64, Int64, Ptr{Float64}), ctx, ptype, 0, length(ids), R))
        end
        ids = [i for i in r.order[r.shard[k]] if r.cfmms[i] isa UniV3]
        isempty(ids) && continue
        cp = Float64[r.cfmms[i].current_price for i in ids]
        lq = reduce(vcat, (Float64.(r.cfmms[i].liquidity) for i in ids))
        chk(ctx, ccall((:cfmm_update_univ3, LIB), Cint,
            (Ptr{Cvoid}, Int64, Int64, Ptr{Float64}, Ptr{Float64}), ctx, 0, length(ids), cp, lq))
    end
end

# Changing the pool set of one context after cfmm_finalize (cfmm_b200.h): pools appended with the
# next insertion indices, pools retired and restored, the current state read back, the appended
# pools folded into the main layout.  R, w: [2m] pool-major; Ai: [2m] 1-based; ptype: 0 / 1 / 2.
append_product!(ctx, R::Vector{Float64}, γ::Vector{Float64}, Ai::Vector{Int64}) =
    chk(ctx, ccall((:cfmm_append_product, LIB), Cint,
        (Ptr{Cvoid}, Int64, Ptr{Float64}, Ptr{Float64}, Ptr{Int64}), ctx, length(γ), R, γ, Ai))
append_geomean!(ctx, R::Vector{Float64}, γ::Vector{Float64}, Ai::Vector{Int64}, w::Vector{Float64}) =
    chk(ctx, ccall((:cfmm_append_geomean, LIB), Cint,
        (Ptr{Cvoid}, Int64, Ptr{Float64}, Ptr{Float64}, Ptr{Int64}, Ptr{Float64}), ctx, length(γ), R, γ, Ai, w))
append_univ3!(ctx, cp::Vector{Float64}, γ::Vector{Float64}, Ai::Vector{Int64}, tick_off::Vector{Int64},
              lower::Vector{Float64}, liq::Vector{Float64}) =
    chk(ctx, ccall((:cfmm_append_univ3, LIB), Cint,
        (Ptr{Cvoid}, Int64, Ptr{Float64}, Ptr{Float64}, Ptr{Int64}, Ptr{Int64}, Ptr{Float64}, Ptr{Float64}),
        ctx, length(cp), cp, γ, Ai, tick_off, lower, liq))
set_active!(ctx, ptype::Integer, first::Integer, active::AbstractVector{Bool}) =
    chk(ctx, ccall((:cfmm_set_active, LIB), Cint, (Ptr{Cvoid}, Cint, Int64, Int64, Ptr{UInt8}),
        ctx, ptype, first, length(active), UInt8.(active)))
function pool_state(ctx, ptype::Integer, first::Integer, count::Integer)
    state = zeros(Float64, ptype == 2 ? count : 2count)
    active = zeros(UInt8, count)
    chk(ctx, ccall((:cfmm_get_pool_state, LIB), Cint,
        (Ptr{Cvoid}, Cint, Int64, Int64, Ptr{Float64}, Ptr{UInt8}), ctx, ptype, first, count, state, active))
    return state, active .!= 0
end
compact!(ctx) = chk(ctx, ccall((:cfmm_compact, LIB), Cint, (Ptr{Cvoid},), ctx))

# Swaps against the device-resident pools (cfmm_quote_swaps / cfmm_execute_swaps).  pools are
# 0-based indices in the type's insertion order; tender is 2 x q (column j = row j's Δ in the
# pool's token order); both return received as 2 x q.  Like the rest of this file, never executed.
function quote_swaps(ctx, ptype::Integer, pools::Vector{Int64}, tender::Matrix{Float64})
    size(tender) == (2, length(pools)) || throw(ArgumentError("tender must be 2 x length(pools)"))
    received = zeros(Float64, 2, length(pools))
    chk(ctx, ccall((:cfmm_quote_swaps, LIB), Cint,
        (Ptr{Cvoid}, Cint, Int64, Ptr{Int64}, Ptr{Float64}, Ptr{Float64}),
        ctx, ptype, length(pools), pools, tender, received))
    return received
end
function execute_swaps!(ctx, ptype::Integer, pools::Vector{Int64}, tender::Matrix{Float64})
    size(tender) == (2, length(pools)) || throw(ArgumentError("tender must be 2 x length(pools)"))
    received = zeros(Float64, 2, length(pools))
    chk(ctx, ccall((:cfmm_execute_swaps, LIB), Cint,
        (Ptr{Cvoid}, Cint, Int64, Ptr{Int64}, Ptr{Float64}, Ptr{Float64}),
        ctx, ptype, length(pools), pools, tender, received))
    return received
end

# Exact-output quotes and order rows with slippage limits (cfmm_quote_swaps_exact_out /
# cfmm_execute_swap_orders).  want / amount are 2 x q as tender above; kind is 0 (exact-in) or 1
# (exact-out) per row; limit is nothing or a length-q vector.  execute_swap_orders! returns
# (paid, received, status).  Like the rest of this file, never executed.
const SWAP_EXACT_IN = 0
const SWAP_EXACT_OUT = 1
const ORDER_FILLED, ORDER_LIMIT, ORDER_UNREACHABLE, ORDER_RETIRED = 0, 1, 2, 3
function quote_swaps_exact_out(ctx, ptype::Integer, pools::Vector{Int64}, want::Matrix{Float64})
    size(want) == (2, length(pools)) || throw(ArgumentError("want must be 2 x length(pools)"))
    tender = zeros(Float64, 2, length(pools))
    chk(ctx, ccall((:cfmm_quote_swaps_exact_out, LIB), Cint,
        (Ptr{Cvoid}, Cint, Int64, Ptr{Int64}, Ptr{Float64}, Ptr{Float64}),
        ctx, ptype, length(pools), pools, want, tender))
    return tender
end
function execute_swap_orders!(ctx, ptype::Integer, pools::Vector{Int64}, kind::Vector{UInt8},
                              amount::Matrix{Float64}, limit::Union{Nothing,Vector{Float64}}=nothing)
    q = length(pools)
    size(amount) == (2, q) || throw(ArgumentError("amount must be 2 x length(pools)"))
    length(kind) == q || throw(ArgumentError("kind must have length(pools) entries"))
    limit === nothing || length(limit) == q || throw(ArgumentError("limit must have length(pools) entries"))
    paid, received, status = zeros(Float64, 2, q), zeros(Float64, 2, q), zeros(UInt8, q)
    chk(ctx, ccall((:cfmm_execute_swap_orders, LIB), Cint,
        (Ptr{Cvoid}, Cint, Int64, Ptr{Int64}, Ptr{UInt8}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64},
         Ptr{Float64}, Ptr{UInt8}),
        ctx, ptype, q, pools, kind, amount, limit === nothing ? C_NULL : limit, paid, received, status))
    return paid, received, status
end

# Multi-hop swap paths (cfmm_quote_paths / cfmm_execute_paths).  Path j is the hops
# hop_off[j]+1 .. hop_off[j+1] of hop_type / hop_pool (hop_off is the 0-based CSR offset vector of
# length q+1; pools are 0-based insertion indices of their type); token_in is 1-based.  Both
# return (hop_tender, hop_received, status).  Like the rest of this file, never executed.
const PATH_MAX_HOPS = 8
function _check_paths(hop_off, hop_type, hop_pool, token_in, kind, amount)
    q = length(hop_off) - 1
    q >= 0 && length(token_in) == length(kind) == length(amount) == q ||
        throw(ArgumentError("hop_off needs q+1 entries, token_in / kind / amount q each"))
    length(hop_type) == length(hop_pool) == hop_off[end] ||
        throw(ArgumentError("hop_type / hop_pool need hop_off[end] entries"))
    return q, Int(hop_off[end])
end
function quote_paths(ctx, hop_off::Vector{Int64}, hop_type::Vector{Cint}, hop_pool::Vector{Int64},
                     token_in::Vector{Int64}, kind::Vector{UInt8}, amount::Vector{Float64})
    q, H = _check_paths(hop_off, hop_type, hop_pool, token_in, kind, amount)
    tender, received, status = zeros(Float64, H), zeros(Float64, H), zeros(UInt8, q)
    chk(ctx, ccall((:cfmm_quote_paths, LIB), Cint,
        (Ptr{Cvoid}, Int64, Ptr{Int64}, Ptr{Cint}, Ptr{Int64}, Ptr{Int64}, Ptr{UInt8}, Ptr{Float64},
         Ptr{Float64}, Ptr{Float64}, Ptr{UInt8}),
        ctx, q, hop_off, hop_type, hop_pool, token_in, kind, amount, tender, received, status))
    return tender, received, status
end
function execute_paths!(ctx, hop_off::Vector{Int64}, hop_type::Vector{Cint}, hop_pool::Vector{Int64},
                        token_in::Vector{Int64}, kind::Vector{UInt8}, amount::Vector{Float64},
                        limit::Union{Nothing,Vector{Float64}}=nothing)
    q, H = _check_paths(hop_off, hop_type, hop_pool, token_in, kind, amount)
    limit === nothing || length(limit) == q || throw(ArgumentError("limit must have q entries"))
    tender, received, status = zeros(Float64, H), zeros(Float64, H), zeros(UInt8, q)
    chk(ctx, ccall((:cfmm_execute_paths, LIB), Cint,
        (Ptr{Cvoid}, Int64, Ptr{Int64}, Ptr{Cint}, Ptr{Int64}, Ptr{Int64}, Ptr{UInt8}, Ptr{Float64},
         Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{UInt8}),
        ctx, q, hop_off, hop_type, hop_pool, token_in, kind, amount, limit === nothing ? C_NULL : limit,
        tender, received, status))
    return tender, received, status
end

# Orders split across every pool of their token pair (cfmm_pair_pools / cfmm_quote_split_orders /
# cfmm_execute_split_orders).  Tokens are 1-based.  pair_pools returns (count, type, pool, active),
# pools 0-based insertion indices of their type, each row's pools after the previous row's.  The
# split calls return (paid, received, price, status, leg_delta, leg_lambda); the legs are 2 x L
# (column = one pool's (Δ, Λ) side), rows after one another in pair_pools order.  Like the rest of
# this file, never executed.
function pair_pools(ctx, token_a::Vector{Int64}, token_b::Vector{Int64})
    q = length(token_a)
    length(token_b) == q || throw(ArgumentError("token_a and token_b need one entry per row"))
    count = zeros(Int64, q)
    chk(ctx, ccall((:cfmm_pair_pools, LIB), Cint,
        (Ptr{Cvoid}, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{Int64}, Int64, Ptr{Cint}, Ptr{Int64}, Ptr{UInt8}),
        ctx, q, token_a, token_b, count, 0, C_NULL, C_NULL, C_NULL))
    L = sum(count; init=0)
    typ, pool, active = zeros(Cint, L), zeros(Int64, L), zeros(UInt8, L)
    L > 0 && chk(ctx, ccall((:cfmm_pair_pools, LIB), Cint,
        (Ptr{Cvoid}, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{Int64}, Int64, Ptr{Cint}, Ptr{Int64}, Ptr{UInt8}),
        ctx, q, token_a, token_b, count, L, typ, pool, active))
    return count, typ, pool, active
end
function _split_orders(fn, ctx, token_in, token_out, kind, amount, limit)
    q = length(token_in)
    length(token_out) == length(kind) == length(amount) == q ||
        throw(ArgumentError("token_in / token_out / kind / amount need one entry per row"))
    limit === nothing || length(limit) == q || throw(ArgumentError("limit must have q entries"))
    L = sum(pair_pools(ctx, token_in, token_out)[1]; init=0)
    paid, received, price, status = zeros(q), zeros(q), zeros(q), zeros(UInt8, q)
    ld, ll = zeros(2, L), zeros(2, L)
    if fn === :quote
        chk(ctx, ccall((:cfmm_quote_split_orders, LIB), Cint,
            (Ptr{Cvoid}, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{UInt8}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64},
             Ptr{Float64}, Ptr{UInt8}, Ptr{Float64}, Ptr{Float64}),
            ctx, q, token_in, token_out, kind, amount, paid, received, price, status, ld, ll))
    else
        chk(ctx, ccall((:cfmm_execute_split_orders, LIB), Cint,
            (Ptr{Cvoid}, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{UInt8}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64},
             Ptr{Float64}, Ptr{Float64}, Ptr{UInt8}, Ptr{Float64}, Ptr{Float64}),
            ctx, q, token_in, token_out, kind, amount, limit === nothing ? C_NULL : limit, paid, received,
            price, status, ld, ll))
    end
    return paid, received, price, status, ld, ll
end
quote_split_orders(ctx, token_in::Vector{Int64}, token_out::Vector{Int64}, kind::Vector{UInt8},
                   amount::Vector{Float64}) = _split_orders(:quote, ctx, token_in, token_out, kind, amount, nothing)
execute_split_orders!(ctx, token_in::Vector{Int64}, token_out::Vector{Int64}, kind::Vector{UInt8},
                      amount::Vector{Float64}, limit::Union{Nothing,Vector{Float64}}=nothing) =
    _split_orders(:execute, ctx, token_in, token_out, kind, amount, limit)

# Orders routed over their pair and the two-hop routes through hub tokens (cfmm_quote_routed_orders /
# cfmm_execute_routed_orders).  Row r's hubs are hubs[hub_off[r]+1 : hub_off[r+1]] (1-based tokens,
# hub_off 0-based offsets, at most 7 per row).  Returns (paid, received, price, status, hub_price,
# hub_surplus, leg_delta, leg_lambda); each row's legs are its pairs' pools in the order (j, i),
# (j, h₁), (h₁, i), (j, h₂), …, in pair_pools order.  Never executed, like the rest of this file.
function _routed_orders(fn, ctx, token_in, token_out, kind, amount, hub_off, hubs, limit)
    q = length(token_in)
    length(token_out) == length(kind) == length(amount) == q && length(hub_off) == q + 1 ||
        throw(ArgumentError("token_in / token_out / kind / amount need q entries, hub_off q + 1"))
    limit === nothing || length(limit) == q || throw(ArgumentError("limit must have q entries"))
    a, b = Int64[], Int64[]
    for r in 1:q
        push!(a, token_in[r]); push!(b, token_out[r])
        for h in hubs[hub_off[r]+1:hub_off[r+1]]
            push!(a, token_in[r], h); push!(b, h, token_out[r])
        end
    end
    L = sum(pair_pools(ctx, a, b)[1]; init=0)
    nh = length(hubs)
    paid, received, price, status = zeros(q), zeros(q), zeros(q), zeros(UInt8, q)
    hp, hs, ld, ll = zeros(nh), zeros(nh), zeros(2, L), zeros(2, L)
    if fn === :quote
        chk(ctx, ccall((:cfmm_quote_routed_orders, LIB), Cint,
            (Ptr{Cvoid}, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{UInt8}, Ptr{Float64}, Ptr{Int64}, Ptr{Int64},
             Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{UInt8}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64},
             Ptr{Float64}),
            ctx, q, token_in, token_out, kind, amount, hub_off, hubs, paid, received, price, status, hp, hs, ld, ll))
    else
        chk(ctx, ccall((:cfmm_execute_routed_orders, LIB), Cint,
            (Ptr{Cvoid}, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{UInt8}, Ptr{Float64}, Ptr{Float64}, Ptr{Int64},
             Ptr{Int64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{UInt8}, Ptr{Float64}, Ptr{Float64},
             Ptr{Float64}, Ptr{Float64}),
            ctx, q, token_in, token_out, kind, amount, limit === nothing ? C_NULL : limit, hub_off, hubs, paid,
            received, price, status, hp, hs, ld, ll))
    end
    return paid, received, price, status, hp, hs, ld, ll
end
quote_routed_orders(ctx, token_in::Vector{Int64}, token_out::Vector{Int64}, kind::Vector{UInt8},
                    amount::Vector{Float64}, hub_off::Vector{Int64}, hubs::Vector{Int64}) =
    _routed_orders(:quote, ctx, token_in, token_out, kind, amount, hub_off, hubs, nothing)
execute_routed_orders!(ctx, token_in::Vector{Int64}, token_out::Vector{Int64}, kind::Vector{UInt8},
                       amount::Vector{Float64}, hub_off::Vector{Int64}, hubs::Vector{Int64},
                       limit::Union{Nothing,Vector{Float64}}=nothing) =
    _routed_orders(:execute, ctx, token_in, token_out, kind, amount, hub_off, hubs, limit)

# Arbitrage cycles through base tokens (cfmm_quote_arbitrage / cfmm_execute_arbitrage /
# cfmm_scan_arbitrage).  Row r runs the cycles from base[r] through other[r] and back, directly and
# through the hubs hubs[hub_off[r]+1 : hub_off[r+1]].  Returns (profit, surplus_in, price, status,
# hub_price, hub_surplus, leg_delta, leg_lambda), legs in the pair order (other, base), (other, h₁),
# (h₁, base), ….  scan_arbitrage returns (found, base, other, hub_off, hubs, profit, price) of the first
# min(found, cap) rows.  Never executed, like the rest of this file.
function _arbitrage(fn, ctx, base, other, hub_off, hubs, min_profit)
    q = length(base)
    length(other) == q && length(hub_off) == q + 1 ||
        throw(ArgumentError("base / other need q entries, hub_off q + 1"))
    min_profit === nothing || length(min_profit) == q || throw(ArgumentError("min_profit must have q entries"))
    a, b = Int64[], Int64[]
    for r in 1:q
        push!(a, other[r]); push!(b, base[r])
        for h in hubs[hub_off[r]+1:hub_off[r+1]]
            push!(a, other[r], h); push!(b, h, base[r])
        end
    end
    L = sum(pair_pools(ctx, a, b)[1]; init=0)
    nh = length(hubs)
    profit, surplus, price, status = zeros(q), zeros(q), zeros(q), zeros(UInt8, q)
    hp, hs, ld, ll = zeros(nh), zeros(nh), zeros(2, L), zeros(2, L)
    if fn === :quote
        chk(ctx, ccall((:cfmm_quote_arbitrage, LIB), Cint,
            (Ptr{Cvoid}, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{Int64}, Ptr{Int64}, Ptr{Float64}, Ptr{Float64},
             Ptr{Float64}, Ptr{UInt8}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}),
            ctx, q, base, other, hub_off, hubs, profit, surplus, price, status, hp, hs, ld, ll))
    else
        chk(ctx, ccall((:cfmm_execute_arbitrage, LIB), Cint,
            (Ptr{Cvoid}, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{Float64}, Ptr{Int64}, Ptr{Int64}, Ptr{Float64},
             Ptr{Float64}, Ptr{Float64}, Ptr{UInt8}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}),
            ctx, q, base, other, min_profit === nothing ? C_NULL : min_profit, hub_off, hubs, profit, surplus,
            price, status, hp, hs, ld, ll))
    end
    return profit, surplus, price, status, hp, hs, ld, ll
end
quote_arbitrage(ctx, base::Vector{Int64}, other::Vector{Int64}, hub_off::Vector{Int64}, hubs::Vector{Int64}) =
    _arbitrage(:quote, ctx, base, other, hub_off, hubs, nothing)
execute_arbitrage!(ctx, base::Vector{Int64}, other::Vector{Int64}, hub_off::Vector{Int64}, hubs::Vector{Int64},
                   min_profit::Union{Nothing,Vector{Float64}}=nothing) =
    _arbitrage(:execute, ctx, base, other, hub_off, hubs, min_profit)

function scan_arbitrage(ctx, base::Vector{Int64}, min_profit::Vector{Float64}, max_hubs::Integer, cap::Integer)
    length(min_profit) == length(base) || throw(ArgumentError("min_profit must have one entry per base token"))
    found = Ref{Int64}(0)
    rb, ro, hc = zeros(Int64, cap), zeros(Int64, cap), zeros(Int64, cap)
    hb, pr, px = zeros(Int64, 7, cap), zeros(cap), zeros(cap)
    chk(ctx, ccall((:cfmm_scan_arbitrage, LIB), Cint,
        (Ptr{Cvoid}, Int64, Ptr{Int64}, Ptr{Float64}, Cint, Int64, Ref{Int64}, Ptr{Int64}, Ptr{Int64}, Ptr{Int64},
         Ptr{Int64}, Ptr{Float64}, Ptr{Float64}),
        ctx, length(base), base, min_profit, max_hubs, cap, found, rb, ro, hc, hb, pr, px))
    n = min(found[], cap)
    hub_off = vcat(0, cumsum(hc[1:n]))
    hubs = reduce(vcat, [hb[1:hc[r], r] for r in 1:n]; init=Int64[])
    return found[], rb[1:n], ro[1:n], hub_off, hubs, pr[1:n], px[1:n]
end

# Hub tokens chosen for order rows (cfmm_choose_order_hubs): up to max_hubs (0..7) common neighbours of
# token_in[r] and token_out[r] per row, ranked by their best single two-hop route; allowed (nothing:
# every token) is a mask over the tokens.  Returns (hub_off, hubs, score, n_eligible); hub_off and hubs
# go to quote_routed_orders / execute_routed_orders! as they are.  Never executed, like the rest of
# this file.
function choose_order_hubs(ctx, token_in::Vector{Int64}, token_out::Vector{Int64}, kind::Vector{UInt8},
                           amount::Vector{Float64}, max_hubs::Integer,
                           allowed::Union{Nothing,Vector{UInt8}}=nothing)
    q = length(token_in)
    length(token_out) == length(kind) == length(amount) == q ||
        throw(ArgumentError("token_in / token_out / kind / amount need q entries"))
    cap = max(q * max_hubs, 1)
    hub_off, hubs, score, n_elig = zeros(Int64, q + 1), zeros(Int64, cap), zeros(cap), zeros(Int64, q)
    chk(ctx, ccall((:cfmm_choose_order_hubs, LIB), Cint,
        (Ptr{Cvoid}, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{UInt8}, Ptr{Float64}, Cint, Ptr{UInt8}, Ptr{Int64},
         Ptr{Int64}, Ptr{Float64}, Ptr{Int64}),
        ctx, q, token_in, token_out, kind, amount, max_hubs, allowed === nothing ? C_NULL : allowed, hub_off,
        hubs, score, n_elig))
    n = hub_off[end]
    return hub_off, hubs[1:n], score[1:n], n_elig
end

# The best path of each order row through allowed tokens (cfmm_find_order_paths): at most max_hops
# (1..8) hops, one pool per hop, every intermediate token t with allowed[t] != 0 (required, one entry
# per token).  Returns (hop_off, hop_type, hop_pool, hop_token, hop_tender, hop_received, value,
# status); hop_off, hop_type and hop_pool go to quote_paths / execute_paths! as they are.  Never
# executed, like the rest of this file.
function find_order_paths(ctx, token_in::Vector{Int64}, token_out::Vector{Int64}, kind::Vector{UInt8},
                          amount::Vector{Float64}, max_hops::Integer, allowed::Vector{UInt8})
    q = length(token_in)
    length(token_out) == length(kind) == length(amount) == q ||
        throw(ArgumentError("token_in / token_out / kind / amount need q entries"))
    cap = max(q * max_hops, 1)
    hop_off, typ, pool, tok = zeros(Int64, q + 1), zeros(Cint, cap), zeros(Int64, cap), zeros(Int64, cap)
    tender, received, value, status = zeros(cap), zeros(cap), zeros(q), zeros(UInt8, q)
    chk(ctx, ccall((:cfmm_find_order_paths, LIB), Cint,
        (Ptr{Cvoid}, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{UInt8}, Ptr{Float64}, Cint, Ptr{UInt8}, Ptr{Int64},
         Ptr{Cint}, Ptr{Int64}, Ptr{Int64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{UInt8}),
        ctx, q, token_in, token_out, kind, amount, max_hops, allowed, hop_off, typ, pool, tok, tender, received,
        value, status))
    n = hop_off[end]
    return hop_off, typ[1:n], pool[1:n], tok[1:n], tender[1:n], received[1:n], value, status
end

# Every token's value against each row's root (cfmm_quote_token_values): kind 0 spends amount[r] of
# root[r], kind 1 receives amount[r] of it; the best walk of at most max_hops (1..8) hops to (kind 0) or
# from (kind 1) every token through tokens t with allowed[t] != 0 (nothing: every token).  value, hops
# and status are n_tokens x q (column r is row r); frontier is max_hops x q, the tokens changed per
# level.  req_row (0-based) / req_token (1-based) name the walks to return, as quote_paths /
# execute_paths! take them.  Never executed, like the rest of this file.
function quote_token_values(ctx, n_tokens::Integer, root::Vector{Int64}, kind::Vector{UInt8},
                            amount::Vector{Float64}, max_hops::Integer, allowed=nothing;
                            req_row::Vector{Int64}=Int64[], req_token::Vector{Int64}=Int64[])
    q, k = length(root), length(req_row)
    length(kind) == length(amount) == q || throw(ArgumentError("root / kind / amount need q entries"))
    length(req_token) == k || throw(ArgumentError("req_row / req_token need one entry per request"))
    value, hops, status = zeros(n_tokens, q), zeros(UInt8, n_tokens, q), zeros(UInt8, n_tokens, q)
    frontier = zeros(Int64, max_hops, q)
    cap = max(k * max_hops, 1)
    hop_off, typ, pool, tok = zeros(Int64, k + 1), zeros(Cint, cap), zeros(Int64, cap), zeros(Int64, cap)
    tender, received, req_status = zeros(cap), zeros(cap), zeros(UInt8, max(k, 1))
    mask = allowed === nothing ? C_NULL : Vector{UInt8}(allowed)
    chk(ctx, ccall((:cfmm_quote_token_values, LIB), Cint,
        (Ptr{Cvoid}, Int64, Ptr{Int64}, Ptr{UInt8}, Ptr{Float64}, Cint, Ptr{UInt8}, Ptr{Float64}, Ptr{UInt8},
         Ptr{UInt8}, Ptr{Int64}, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{Int64}, Ptr{Cint}, Ptr{Int64}, Ptr{Int64},
         Ptr{Float64}, Ptr{Float64}, Ptr{UInt8}),
        ctx, q, root, kind, amount, max_hops, mask, value, hops, status, frontier, k, req_row, req_token,
        hop_off, typ, pool, tok, tender, received, req_status))
    n = hop_off[end]
    return (value=value, hops=hops, status=status, frontier=frontier, hop_off=hop_off, hop_type=typ[1:n],
            hop_pool=pool[1:n], hop_token=tok[1:n], hop_tender=tender[1:n], hop_received=received[1:n],
            req_status=req_status[1:k])
end

# find_order_paths net of a per-hop cost (cfmm_find_order_paths_net): hop_cost[r] is row r's cost of one
# hop in the token it settles in (token_out kind 0, token_in kind 1), >= 0, Inf allowed.  Among
# max_hops = 1..max_hops, the filled result whose value net of the costs is best (the larger on a tie).
# Returns find_order_paths' tuple and net.  Never executed, like the rest of this file.
function find_order_paths_net(ctx, token_in::Vector{Int64}, token_out::Vector{Int64}, kind::Vector{UInt8},
                              amount::Vector{Float64}, max_hops::Integer, allowed::Vector{UInt8},
                              hop_cost::Vector{Float64})
    q = length(token_in)
    length(token_out) == length(kind) == length(amount) == length(hop_cost) == q ||
        throw(ArgumentError("token_in / token_out / kind / amount / hop_cost need q entries"))
    cap = max(q * max_hops, 1)
    hop_off, typ, pool, tok = zeros(Int64, q + 1), zeros(Cint, cap), zeros(Int64, cap), zeros(Int64, cap)
    tender, received, value, status, net = zeros(cap), zeros(cap), zeros(q), zeros(UInt8, q), zeros(q)
    chk(ctx, ccall((:cfmm_find_order_paths_net, LIB), Cint,
        (Ptr{Cvoid}, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{UInt8}, Ptr{Float64}, Cint, Ptr{UInt8}, Ptr{Float64},
         Ptr{Int64}, Ptr{Cint}, Ptr{Int64}, Ptr{Int64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{UInt8},
         Ptr{Float64}),
        ctx, q, token_in, token_out, kind, amount, max_hops, allowed, hop_cost, hop_off, typ, pool, tok, tender,
        received, value, status, net))
    n = hop_off[end]
    return hop_off, typ[1:n], pool[1:n], tok[1:n], tender[1:n], received[1:n], value, status, net
end

# quote_token_values net of a per-hop cost (cfmm_quote_token_values_net): hop_cost[t] is the cost of
# one hop in units of token t (n_tokens entries, >= 0, Inf allowed).  Per (row, token), among max_hops =
# 1..max_hops the filled result whose value net of the costs is best (the larger on a tie); the requested
# walks are the selected ones.  Returns quote_token_values' named tuple with net (n_tokens x q).  Never
# executed, like the rest of this file.
function quote_token_values_net(ctx, n_tokens::Integer, root::Vector{Int64}, kind::Vector{UInt8},
                                amount::Vector{Float64}, max_hops::Integer, hop_cost::Vector{Float64},
                                allowed=nothing; req_row::Vector{Int64}=Int64[], req_token::Vector{Int64}=Int64[])
    q, k = length(root), length(req_row)
    length(kind) == length(amount) == q || throw(ArgumentError("root / kind / amount need q entries"))
    length(hop_cost) == n_tokens || throw(ArgumentError("hop_cost needs one entry per token"))
    length(req_token) == k || throw(ArgumentError("req_row / req_token need one entry per request"))
    value, hops, status = zeros(n_tokens, q), zeros(UInt8, n_tokens, q), zeros(UInt8, n_tokens, q)
    net, frontier = zeros(n_tokens, q), zeros(Int64, max_hops, q)
    cap = max(k * max_hops, 1)
    hop_off, typ, pool, tok = zeros(Int64, k + 1), zeros(Cint, cap), zeros(Int64, cap), zeros(Int64, cap)
    tender, received, req_status = zeros(cap), zeros(cap), zeros(UInt8, max(k, 1))
    mask = allowed === nothing ? C_NULL : Vector{UInt8}(allowed)
    chk(ctx, ccall((:cfmm_quote_token_values_net, LIB), Cint,
        (Ptr{Cvoid}, Int64, Ptr{Int64}, Ptr{UInt8}, Ptr{Float64}, Cint, Ptr{UInt8}, Ptr{Float64}, Ptr{Float64},
         Ptr{UInt8}, Ptr{UInt8}, Ptr{Float64}, Ptr{Int64}, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{Int64}, Ptr{Cint},
         Ptr{Int64}, Ptr{Int64}, Ptr{Float64}, Ptr{Float64}, Ptr{UInt8}),
        ctx, q, root, kind, amount, max_hops, mask, hop_cost, value, hops, status, net, frontier, k, req_row,
        req_token, hop_off, typ, pool, tok, tender, received, req_status))
    n = hop_off[end]
    return (value=value, hops=hops, status=status, net=net, frontier=frontier, hop_off=hop_off,
            hop_type=typ[1:n], hop_pool=pool[1:n], hop_token=tok[1:n], hop_tender=tender[1:n],
            hop_received=received[1:n], req_status=req_status[1:k])
end

# Orders over every pool among allowed tokens (cfmm_quote_subgraph_swap_orders /
# cfmm_execute_subgraph_swap_orders): row r sells amount[r] of token_in[r] for token_out[r] (kind 0,
# exact-in) or buys amount[r] of token_out[r] paying in token_in[r] (kind 1, exact-out) over every pool
# among the two and the tokens t with allowed[t] != 0 (required, one entry per token, at most 256 besides
# the row's two), route! over those pools, one dual solve per row.  kind = nothing: every row exact-in;
# limit: the minimum received (exact-in) or the maximum paid (exact-out).  opts = nothing: the defaults.
# Returns a
# NamedTuple of the per-row outputs, the token CSR (tok_off, token, nu, psi) and the legs CSR
# (leg_off, leg_type, leg_pool, leg_delta / leg_lambda as 2 x L).  Never executed, like the rest of
# this file.
struct SubgraphOpts
    max_iter::Cint
    max_fun::Cint
    rtol::Float64
    factr::Float64
end
struct SubgraphOut
    paid::Ptr{Float64}; received::Ptr{Float64}; status::Ptr{UInt8}
    solver_status::Ptr{Cint}; iterations::Ptr{Cint}; fun_evals::Ptr{Cint}; merit::Ptr{Float64}
    tok_off::Ptr{Int64}; tok_cap::Int64; token::Ptr{Int64}; nu::Ptr{Float64}; psi::Ptr{Float64}
    leg_off::Ptr{Int64}; leg_cap::Int64; leg_type::Ptr{Cint}; leg_pool::Ptr{Int64}
    leg_delta::Ptr{Float64}; leg_lambda::Ptr{Float64}
end
# Per-row masks (cfmm_*_rows): allowed may instead be one Vector of 1-based tokens per row (for example
# choose_hubs' lists); each row then runs over its own list.
_row_csr(lists) = (Int64[0; cumsum(length.(lists))], Int64.(reduce(vcat, lists; init=Int64[])))
function _subgraph_orders(ctx, execute::Bool, token_in::Vector{Int64}, token_out::Vector{Int64},
                          amount::Vector{Float64}, allowed, limit, opts, kind=nothing)
    allowed isa AbstractVector{<:AbstractVector} &&
        return _subgraph_orders_rows(ctx, execute, token_in, token_out, amount, _row_csr(allowed)..., limit, opts,
                                     kind)
    q = length(token_in)
    length(token_out) == length(amount) == q || throw(ArgumentError("token_in / token_out / amount need q entries"))
    limit === nothing || length(limit) == q || throw(ArgumentError("limit needs q entries"))
    k = kind === nothing ? C_NULL : (kind isa Integer ? fill(UInt8(kind), q) : Vector{UInt8}(kind))
    k === C_NULL || length(k) == q || throw(ArgumentError("kind needs q entries"))
    o = opts === nothing ? nothing : Ref(opts)
    tok_off, leg_off = zeros(Int64, q + 1), zeros(Int64, q + 1)
    sizes = Ref(SubgraphOut(C_NULL, C_NULL, C_NULL, C_NULL, C_NULL, C_NULL, C_NULL, pointer(tok_off), 0, C_NULL,
                            C_NULL, C_NULL, pointer(leg_off), 0, C_NULL, C_NULL, C_NULL, C_NULL))
    GC.@preserve tok_off leg_off k chk(ctx, ccall((:cfmm_quote_subgraph_swap_orders, LIB), Cint,
        (Ptr{Cvoid}, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{UInt8}, Ptr{Float64}, Ptr{UInt8}, Ptr{SubgraphOpts},
         Ptr{SubgraphOut}),
        ctx, q, token_in, token_out, k, amount, allowed, o === nothing ? C_NULL : o, sizes))
    NT, L = tok_off[end], leg_off[end]
    paid, received, merit, status = zeros(q), zeros(q), zeros(q), zeros(UInt8, q)
    sst, iters, fev = zeros(Cint, q), zeros(Cint, q), zeros(Cint, q)
    token, nu, psi = zeros(Int64, max(NT, 1)), zeros(max(NT, 1)), zeros(max(NT, 1))
    ltype, lpool, ld, ll = zeros(Cint, max(L, 1)), zeros(Int64, max(L, 1)), zeros(2, max(L, 1)), zeros(2, max(L, 1))
    GC.@preserve paid received merit status sst iters fev tok_off token nu psi leg_off ltype lpool ld ll k begin
        out = Ref(SubgraphOut(pointer(paid), pointer(received), pointer(status), pointer(sst), pointer(iters),
                              pointer(fev), pointer(merit), pointer(tok_off), NT, pointer(token), pointer(nu),
                              pointer(psi), pointer(leg_off), L, pointer(ltype), pointer(lpool), pointer(ld),
                              pointer(ll)))
        if execute
            chk(ctx, ccall((:cfmm_execute_subgraph_swap_orders, LIB), Cint,
                (Ptr{Cvoid}, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{UInt8}, Ptr{Float64}, Ptr{Float64}, Ptr{UInt8},
                 Ptr{SubgraphOpts}, Ptr{SubgraphOut}),
                ctx, q, token_in, token_out, k, amount, limit === nothing ? C_NULL : limit, allowed,
                o === nothing ? C_NULL : o, out))
        else
            chk(ctx, ccall((:cfmm_quote_subgraph_swap_orders, LIB), Cint,
                (Ptr{Cvoid}, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{UInt8}, Ptr{Float64}, Ptr{UInt8}, Ptr{SubgraphOpts},
                 Ptr{SubgraphOut}),
                ctx, q, token_in, token_out, k, amount, allowed, o === nothing ? C_NULL : o, out))
        end
    end
    return (paid=paid, received=received, status=status, solver_status=sst, iterations=iters, fun_evals=fev,
            merit=merit, tok_off=tok_off, token=token[1:NT], nu=nu[1:NT], psi=psi[1:NT], leg_off=leg_off,
            leg_type=ltype[1:L], leg_pool=lpool[1:L], leg_delta=ld[:, 1:L], leg_lambda=ll[:, 1:L])
end
function _subgraph_orders_rows(ctx, execute::Bool, token_in::Vector{Int64}, token_out::Vector{Int64},
                               amount::Vector{Float64}, allow_off::Vector{Int64}, allow_token::Vector{Int64}, limit,
                               opts, kind)
    q = length(token_in)
    length(token_out) == length(amount) == q || throw(ArgumentError("token_in / token_out / amount need q entries"))
    length(allow_off) == q + 1 || throw(ArgumentError("allowed needs one token list per row"))
    k = kind === nothing ? C_NULL : (kind isa Integer ? fill(UInt8(kind), q) : Vector{UInt8}(kind))
    o = opts === nothing ? nothing : Ref(opts)
    argq = (Ptr{Cvoid}, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{UInt8}, Ptr{Float64}, Ptr{Int64}, Ptr{Int64},
            Ptr{SubgraphOpts}, Ptr{SubgraphOut})
    tok_off, leg_off = zeros(Int64, q + 1), zeros(Int64, q + 1)
    sizes = Ref(SubgraphOut(C_NULL, C_NULL, C_NULL, C_NULL, C_NULL, C_NULL, C_NULL, pointer(tok_off), 0, C_NULL,
                            C_NULL, C_NULL, pointer(leg_off), 0, C_NULL, C_NULL, C_NULL, C_NULL))
    GC.@preserve tok_off leg_off k chk(ctx, ccall((:cfmm_quote_subgraph_swap_orders_rows, LIB), Cint, argq, ctx, q,
                                                 token_in, token_out, k, amount, allow_off, allow_token,
                                                 o === nothing ? C_NULL : o, sizes))
    NT, L = tok_off[end], leg_off[end]
    paid, received, merit, status = zeros(q), zeros(q), zeros(q), zeros(UInt8, q)
    sst, iters, fev = zeros(Cint, q), zeros(Cint, q), zeros(Cint, q)
    token, nu, psi = zeros(Int64, max(NT, 1)), zeros(max(NT, 1)), zeros(max(NT, 1))
    ltype, lpool, ld, ll = zeros(Cint, max(L, 1)), zeros(Int64, max(L, 1)), zeros(2, max(L, 1)), zeros(2, max(L, 1))
    GC.@preserve paid received merit status sst iters fev tok_off token nu psi leg_off ltype lpool ld ll k begin
        out = Ref(SubgraphOut(pointer(paid), pointer(received), pointer(status), pointer(sst), pointer(iters),
                              pointer(fev), pointer(merit), pointer(tok_off), NT, pointer(token), pointer(nu),
                              pointer(psi), pointer(leg_off), L, pointer(ltype), pointer(lpool), pointer(ld),
                              pointer(ll)))
        if execute
            chk(ctx, ccall((:cfmm_execute_subgraph_swap_orders_rows, LIB), Cint,
                (Ptr{Cvoid}, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{UInt8}, Ptr{Float64}, Ptr{Float64}, Ptr{Int64},
                 Ptr{Int64}, Ptr{SubgraphOpts}, Ptr{SubgraphOut}),
                ctx, q, token_in, token_out, k, amount, limit === nothing ? C_NULL : limit, allow_off, allow_token,
                o === nothing ? C_NULL : o, out))
        else
            chk(ctx, ccall((:cfmm_quote_subgraph_swap_orders_rows, LIB), Cint, argq, ctx, q, token_in, token_out, k,
                           amount, allow_off, allow_token, o === nothing ? C_NULL : o, out))
        end
    end
    return (paid=paid, received=received, status=status, solver_status=sst, iterations=iters, fun_evals=fev,
            merit=merit, tok_off=tok_off, token=token[1:NT], nu=nu[1:NT], psi=psi[1:NT], leg_off=leg_off,
            leg_type=ltype[1:L], leg_pool=lpool[1:L], leg_delta=ld[:, 1:L], leg_lambda=ll[:, 1:L])
end
quote_subgraph_orders(ctx, token_in, token_out, amount, allowed; opts=nothing, kind=nothing) =
    _subgraph_orders(ctx, false, token_in, token_out, amount, allowed, nothing, opts, kind)
execute_subgraph_orders!(ctx, token_in, token_out, amount, allowed; limit=nothing, opts=nothing, kind=nothing) =
    _subgraph_orders(ctx, true, token_in, token_out, amount, allowed, limit, opts, kind)

# Token baskets over every pool among allowed tokens (cfmm_quote_basket_orders /
# cfmm_execute_basket_orders): row r sells basket_amount[k] of basket_token[k] for k in
# basket_off[r]+1 .. basket_off[r+1] (1 to 16 distinct tokens, none of them token_out[r]; basket_off is
# 0-based, q + 1 entries) for token_out[r], route! with BasketLiquidation over those pools.  Returns the
# NamedTuple of _subgraph_orders with paid per basket entry.  The output struct has SubgraphOut's layout
# (cfmm_basket_out).  entry_kind (nothing: every entry sold) is one UInt8 per basket entry, 0 sold or 1
# bought, and selects cfmm_quote/execute_basket_swap_orders.  Never executed, like the rest of this file.
function _basket_orders(ctx, execute::Bool, token_out::Vector{Int64}, basket_off::Vector{Int64},
                        basket_token::Vector{Int64}, basket_amount::Vector{Float64}, allowed, limit,
                        opts, entry_kind=nothing)
    rows = allowed isa AbstractVector{<:AbstractVector}
    aoff, atok = rows ? _row_csr(allowed) : (Int64[], Int64[])
    q = length(token_out)
    length(basket_off) == q + 1 || throw(ArgumentError("basket_off needs q + 1 entries"))
    NE = basket_off[end]
    length(basket_token) == length(basket_amount) == NE ||
        throw(ArgumentError("basket_token / basket_amount need basket_off[end] entries"))
    limit === nothing || length(limit) == q || throw(ArgumentError("limit needs q entries"))
    entry_kind === nothing || length(entry_kind) == NE ||
        throw(ArgumentError("entry_kind needs basket_off[end] entries"))
    o = opts === nothing ? nothing : Ref(opts)
    argt = (Ptr{Cvoid}, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{Int64}, Ptr{Float64}, Ptr{UInt8}, Ptr{SubgraphOpts},
            Ptr{SubgraphOut})
    argk = (Ptr{Cvoid}, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{Int64}, Ptr{UInt8}, Ptr{Float64}, Ptr{UInt8},
            Ptr{SubgraphOpts}, Ptr{SubgraphOut})
    argr = (Ptr{Cvoid}, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{Int64}, Ptr{UInt8}, Ptr{Float64}, Ptr{Int64}, Ptr{Int64},
            Ptr{SubgraphOpts}, Ptr{SubgraphOut})
    ek = entry_kind === nothing ? C_NULL : entry_kind
    quote_call(out) = rows ?
        ccall((:cfmm_quote_basket_swap_orders_rows, LIB), Cint, argr, ctx, q, token_out, basket_off, basket_token,
              ek, basket_amount, aoff, atok, o === nothing ? C_NULL : o, out) :
        entry_kind === nothing ?
        ccall((:cfmm_quote_basket_orders, LIB), Cint, argt, ctx, q, token_out, basket_off, basket_token,
              basket_amount, allowed, o === nothing ? C_NULL : o, out) :
        ccall((:cfmm_quote_basket_swap_orders, LIB), Cint, argk, ctx, q, token_out, basket_off, basket_token,
              entry_kind, basket_amount, allowed, o === nothing ? C_NULL : o, out)
    tok_off, leg_off = zeros(Int64, q + 1), zeros(Int64, q + 1)
    sizes = Ref(SubgraphOut(C_NULL, C_NULL, C_NULL, C_NULL, C_NULL, C_NULL, C_NULL, pointer(tok_off), 0, C_NULL,
                            C_NULL, C_NULL, pointer(leg_off), 0, C_NULL, C_NULL, C_NULL, C_NULL))
    GC.@preserve tok_off leg_off chk(ctx, quote_call(sizes))
    NT, L = tok_off[end], leg_off[end]
    paid, received, merit, status = zeros(max(NE, 1)), zeros(q), zeros(q), zeros(UInt8, q)
    sst, iters, fev = zeros(Cint, q), zeros(Cint, q), zeros(Cint, q)
    token, nu, psi = zeros(Int64, max(NT, 1)), zeros(max(NT, 1)), zeros(max(NT, 1))
    ltype, lpool, ld, ll = zeros(Cint, max(L, 1)), zeros(Int64, max(L, 1)), zeros(2, max(L, 1)), zeros(2, max(L, 1))
    GC.@preserve paid received merit status sst iters fev tok_off token nu psi leg_off ltype lpool ld ll begin
        out = Ref(SubgraphOut(pointer(paid), pointer(received), pointer(status), pointer(sst), pointer(iters),
                              pointer(fev), pointer(merit), pointer(tok_off), NT, pointer(token), pointer(nu),
                              pointer(psi), pointer(leg_off), L, pointer(ltype), pointer(lpool), pointer(ld),
                              pointer(ll)))
        if execute && rows
            chk(ctx, ccall((:cfmm_execute_basket_swap_orders_rows, LIB), Cint,
                (Ptr{Cvoid}, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{Int64}, Ptr{UInt8}, Ptr{Float64}, Ptr{Float64},
                 Ptr{Int64}, Ptr{Int64}, Ptr{SubgraphOpts}, Ptr{SubgraphOut}),
                ctx, q, token_out, basket_off, basket_token, ek, basket_amount,
                limit === nothing ? C_NULL : limit, aoff, atok, o === nothing ? C_NULL : o, out))
        elseif execute && entry_kind !== nothing
            chk(ctx, ccall((:cfmm_execute_basket_swap_orders, LIB), Cint,
                (Ptr{Cvoid}, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{Int64}, Ptr{UInt8}, Ptr{Float64}, Ptr{Float64},
                 Ptr{UInt8}, Ptr{SubgraphOpts}, Ptr{SubgraphOut}),
                ctx, q, token_out, basket_off, basket_token, entry_kind, basket_amount,
                limit === nothing ? C_NULL : limit, allowed, o === nothing ? C_NULL : o, out))
        elseif execute
            chk(ctx, ccall((:cfmm_execute_basket_orders, LIB), Cint,
                (Ptr{Cvoid}, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{Int64}, Ptr{Float64}, Ptr{Float64}, Ptr{UInt8},
                 Ptr{SubgraphOpts}, Ptr{SubgraphOut}),
                ctx, q, token_out, basket_off, basket_token, basket_amount, limit === nothing ? C_NULL : limit,
                allowed, o === nothing ? C_NULL : o, out))
        else
            chk(ctx, quote_call(out))
        end
    end
    return (paid=paid[1:NE], received=received, status=status, solver_status=sst, iterations=iters,
            fun_evals=fev, merit=merit, tok_off=tok_off, token=token[1:NT], nu=nu[1:NT], psi=psi[1:NT],
            leg_off=leg_off, leg_type=ltype[1:L], leg_pool=lpool[1:L], leg_delta=ld[:, 1:L], leg_lambda=ll[:, 1:L])
end
quote_basket_orders(ctx, token_out, basket_off, basket_token, basket_amount, allowed; opts=nothing) =
    _basket_orders(ctx, false, token_out, basket_off, basket_token, basket_amount, allowed, nothing, opts)
execute_basket_orders!(ctx, token_out, basket_off, basket_token, basket_amount, allowed; limit=nothing,
                       opts=nothing) =
    _basket_orders(ctx, true, token_out, basket_off, basket_token, basket_amount, allowed, limit, opts)
# Baskets bought and sold together (cfmm_quote/execute_basket_swap_orders): entry_kind[k] is 0 when entry k
# is sold (up to basket_amount[k]) and 1 when it is bought (at least basket_amount[k]); a row settles in
# token_out[r], and limit[r] is its minimum net of token_out (negative or -Inf allowed on a buy row).
quote_basket_swap_orders(ctx, token_out, basket_off, basket_token, entry_kind, basket_amount, allowed;
                         opts=nothing) =
    _basket_orders(ctx, false, token_out, basket_off, basket_token, basket_amount, allowed, nothing, opts,
                   entry_kind)
execute_basket_swap_orders!(ctx, token_out, basket_off, basket_token, entry_kind, basket_amount, allowed;
                            limit=nothing, opts=nothing) =
    _basket_orders(ctx, true, token_out, basket_off, basket_token, basket_amount, allowed, limit, opts, entry_kind)

# Arbitrage against external prices (cfmm_quote_price_arbitrage / cfmm_execute_price_arbitrage): price is
# n_A x q (column r = row r's prices of the allowed tokens, ascending; 0 leaves a token out), and each
# row maximises price'Ψ with Ψ >= 0 over the pools among its priced tokens (LinearNonnegative).
# min_profit (nothing: none) is one minimum profit per row.  Returns the NamedTuple of _subgraph_orders
# with profit for paid and received.  Never executed, like the rest of this file.
struct PriceArbOut
    profit::Ptr{Float64}; status::Ptr{UInt8}
    solver_status::Ptr{Cint}; iterations::Ptr{Cint}; fun_evals::Ptr{Cint}; merit::Ptr{Float64}
    tok_off::Ptr{Int64}; tok_cap::Int64; token::Ptr{Int64}; nu::Ptr{Float64}; psi::Ptr{Float64}
    leg_off::Ptr{Int64}; leg_cap::Int64; leg_type::Ptr{Cint}; leg_pool::Ptr{Int64}
    leg_delta::Ptr{Float64}; leg_lambda::Ptr{Float64}
end
function _price_arbitrage(ctx, execute::Bool, price::Matrix{Float64}, allowed::Vector{UInt8}, min_profit, opts)
    q = size(price, 2)
    size(price, 1) == count(!=(0), allowed) || throw(ArgumentError("price needs one row per allowed token"))
    min_profit === nothing || length(min_profit) == q || throw(ArgumentError("min_profit needs q entries"))
    o = opts === nothing ? nothing : Ref(opts)
    argq = (Ptr{Cvoid}, Int64, Ptr{Float64}, Ptr{UInt8}, Ptr{SubgraphOpts}, Ptr{PriceArbOut})
    tok_off, leg_off = zeros(Int64, q + 1), zeros(Int64, q + 1)
    sizes = Ref(PriceArbOut(C_NULL, C_NULL, C_NULL, C_NULL, C_NULL, C_NULL, pointer(tok_off), 0, C_NULL, C_NULL,
                            C_NULL, pointer(leg_off), 0, C_NULL, C_NULL, C_NULL, C_NULL))
    GC.@preserve tok_off leg_off chk(ctx, ccall((:cfmm_quote_price_arbitrage, LIB), Cint, argq, ctx, q, price,
                                               allowed, o === nothing ? C_NULL : o, sizes))
    NT, L = tok_off[end], leg_off[end]
    profit, merit, status = zeros(q), zeros(q), zeros(UInt8, q)
    sst, iters, fev = zeros(Cint, q), zeros(Cint, q), zeros(Cint, q)
    token, nu, psi = zeros(Int64, max(NT, 1)), zeros(max(NT, 1)), zeros(max(NT, 1))
    ltype, lpool, ld, ll = zeros(Cint, max(L, 1)), zeros(Int64, max(L, 1)), zeros(2, max(L, 1)), zeros(2, max(L, 1))
    GC.@preserve profit merit status sst iters fev tok_off token nu psi leg_off ltype lpool ld ll begin
        out = Ref(PriceArbOut(pointer(profit), pointer(status), pointer(sst), pointer(iters), pointer(fev),
                              pointer(merit), pointer(tok_off), NT, pointer(token), pointer(nu), pointer(psi),
                              pointer(leg_off), L, pointer(ltype), pointer(lpool), pointer(ld), pointer(ll)))
        if execute
            chk(ctx, ccall((:cfmm_execute_price_arbitrage, LIB), Cint,
                (Ptr{Cvoid}, Int64, Ptr{Float64}, Ptr{Float64}, Ptr{UInt8}, Ptr{SubgraphOpts}, Ptr{PriceArbOut}),
                ctx, q, price, min_profit === nothing ? C_NULL : min_profit, allowed, o === nothing ? C_NULL : o,
                out))
        else
            chk(ctx, ccall((:cfmm_quote_price_arbitrage, LIB), Cint, argq, ctx, q, price, allowed,
                           o === nothing ? C_NULL : o, out))
        end
    end
    return (profit=profit, status=status, solver_status=sst, iterations=iters, fun_evals=fev, merit=merit,
            tok_off=tok_off, token=token[1:NT], nu=nu[1:NT], psi=psi[1:NT], leg_off=leg_off, leg_type=ltype[1:L],
            leg_pool=lpool[1:L], leg_delta=ld[:, 1:L], leg_lambda=ll[:, 1:L])
end
quote_price_arbitrage(ctx, price, allowed; opts=nothing) =
    _price_arbitrage(ctx, false, price, allowed, nothing, opts)
execute_price_arbitrage!(ctx, price, allowed; min_profit=nothing, opts=nothing) =
    _price_arbitrage(ctx, true, price, allowed, min_profit, opts)

# Arbitrage from inventory (cfmm_quote_price_arbitrage_rows / cfmm_execute_price_arbitrage_rows): row r
# lists allow_token[allow_off[r]+1 : allow_off[r+1]] (1-based tokens, any order), with price and holding
# (nothing: none held) aligned with allow_token; each row maximises price'Ψ with Ψ + holding >= 0 over the
# pools among its tokens.  opts is a PriceArbOpts (atol: the absolute stop).  Returns _price_arbitrage's
# NamedTuple.  Never executed, like the rest of this file.
struct PriceArbOpts
    max_iter::Cint; max_fun::Cint; rtol::Float64; factr::Float64; atol::Float64
end
function _price_arbitrage_rows(ctx, execute::Bool, allow_off::Vector{Int64}, allow_token::Vector{Int64},
                               price::Vector{Float64}, holding, min_profit, opts)
    q = length(allow_off) - 1
    length(price) == length(allow_token) || throw(ArgumentError("price needs one entry per listed token"))
    holding === nothing || length(holding) == length(allow_token) ||
        throw(ArgumentError("holding needs one entry per listed token"))
    min_profit === nothing || length(min_profit) == q || throw(ArgumentError("min_profit needs q entries"))
    o = opts === nothing ? nothing : Ref(opts)
    h = holding === nothing ? C_NULL : holding
    argq = (Ptr{Cvoid}, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{Float64}, Ptr{Float64}, Ptr{PriceArbOpts},
            Ptr{PriceArbOut})
    tok_off, leg_off = zeros(Int64, q + 1), zeros(Int64, q + 1)
    sizes = Ref(PriceArbOut(C_NULL, C_NULL, C_NULL, C_NULL, C_NULL, C_NULL, pointer(tok_off), 0, C_NULL, C_NULL,
                            C_NULL, pointer(leg_off), 0, C_NULL, C_NULL, C_NULL, C_NULL))
    GC.@preserve tok_off leg_off chk(ctx, ccall((:cfmm_quote_price_arbitrage_rows, LIB), Cint, argq, ctx, q,
                                               allow_off, allow_token, price, h, o === nothing ? C_NULL : o, sizes))
    NT, L = tok_off[end], leg_off[end]
    profit, merit, status = zeros(q), zeros(q), zeros(UInt8, q)
    sst, iters, fev = zeros(Cint, q), zeros(Cint, q), zeros(Cint, q)
    token, nu, psi = zeros(Int64, max(NT, 1)), zeros(max(NT, 1)), zeros(max(NT, 1))
    ltype, lpool, ld, ll = zeros(Cint, max(L, 1)), zeros(Int64, max(L, 1)), zeros(2, max(L, 1)), zeros(2, max(L, 1))
    GC.@preserve profit merit status sst iters fev tok_off token nu psi leg_off ltype lpool ld ll begin
        out = Ref(PriceArbOut(pointer(profit), pointer(status), pointer(sst), pointer(iters), pointer(fev),
                              pointer(merit), pointer(tok_off), NT, pointer(token), pointer(nu), pointer(psi),
                              pointer(leg_off), L, pointer(ltype), pointer(lpool), pointer(ld), pointer(ll)))
        if execute
            chk(ctx, ccall((:cfmm_execute_price_arbitrage_rows, LIB), Cint,
                (Ptr{Cvoid}, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64},
                 Ptr{PriceArbOpts}, Ptr{PriceArbOut}),
                ctx, q, allow_off, allow_token, price, h, min_profit === nothing ? C_NULL : min_profit,
                o === nothing ? C_NULL : o, out))
        else
            chk(ctx, ccall((:cfmm_quote_price_arbitrage_rows, LIB), Cint, argq, ctx, q, allow_off, allow_token, price,
                           h, o === nothing ? C_NULL : o, out))
        end
    end
    return (profit=profit, status=status, solver_status=sst, iterations=iters, fun_evals=fev, merit=merit,
            tok_off=tok_off, token=token[1:NT], nu=nu[1:NT], psi=psi[1:NT], leg_off=leg_off, leg_type=ltype[1:L],
            leg_pool=lpool[1:L], leg_delta=ld[:, 1:L], leg_lambda=ll[:, 1:L])
end
quote_price_arbitrage_rows(ctx, allow_off, allow_token, price; holding=nothing, opts=nothing) =
    _price_arbitrage_rows(ctx, false, allow_off, allow_token, price, holding, nothing, opts)
execute_price_arbitrage_rows!(ctx, allow_off, allow_token, price; holding=nothing, min_profit=nothing, opts=nothing) =
    _price_arbitrage_rows(ctx, true, allow_off, allow_token, price, holding, min_profit, opts)

# Limit orders with partial fills (cfmm_quote_limit_orders / cfmm_execute_limit_orders): the rows of
# _basket_orders, with limit_price[k] the least token_out[r] per unit of basket_token[k] at the margin
# (finite, >= 0); an entry sells up to basket_amount[k] while the pools pay at least that.  min_received
# (nothing: none) is one minimum received per row.  Returns the NamedTuple of _basket_orders plus surplus
# (received − Σ limit·paid, per row).  Never executed, like the rest of this file.
struct LimitOut
    paid::Ptr{Float64}; received::Ptr{Float64}; status::Ptr{UInt8}
    solver_status::Ptr{Cint}; iterations::Ptr{Cint}; fun_evals::Ptr{Cint}; merit::Ptr{Float64}
    tok_off::Ptr{Int64}; tok_cap::Int64; token::Ptr{Int64}; nu::Ptr{Float64}; psi::Ptr{Float64}
    leg_off::Ptr{Int64}; leg_cap::Int64; leg_type::Ptr{Cint}; leg_pool::Ptr{Int64}
    leg_delta::Ptr{Float64}; leg_lambda::Ptr{Float64}; surplus::Ptr{Float64}
end
function _limit_orders(ctx, execute::Bool, token_out::Vector{Int64}, basket_off::Vector{Int64},
                       basket_token::Vector{Int64}, basket_amount::Vector{Float64}, limit_price::Vector{Float64},
                       allowed, min_received, opts)
    rows = allowed isa AbstractVector{<:AbstractVector}
    aoff, atok = rows ? _row_csr(allowed) : (Int64[], Int64[])
    q = length(token_out)
    length(basket_off) == q + 1 || throw(ArgumentError("basket_off needs q + 1 entries"))
    NE = basket_off[end]
    length(basket_token) == length(basket_amount) == length(limit_price) == NE ||
        throw(ArgumentError("basket_token / basket_amount / limit_price need basket_off[end] entries"))
    min_received === nothing || length(min_received) == q || throw(ArgumentError("min_received needs q entries"))
    o = opts === nothing ? nothing : Ref(opts)
    argq = (Ptr{Cvoid}, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{Int64}, Ptr{Float64}, Ptr{Float64}, Ptr{UInt8},
            Ptr{SubgraphOpts}, Ptr{LimitOut})
    tok_off, leg_off = zeros(Int64, q + 1), zeros(Int64, q + 1)
    sizes = Ref(LimitOut(C_NULL, C_NULL, C_NULL, C_NULL, C_NULL, C_NULL, C_NULL, pointer(tok_off), 0, C_NULL,
                         C_NULL, C_NULL, pointer(leg_off), 0, C_NULL, C_NULL, C_NULL, C_NULL, C_NULL))
    argr = (Ptr{Cvoid}, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{Int64}, Ptr{Float64}, Ptr{Float64}, Ptr{Int64},
            Ptr{Int64}, Ptr{SubgraphOpts}, Ptr{LimitOut})
    quote_call(out) = rows ?
        ccall((:cfmm_quote_limit_orders_rows, LIB), Cint, argr, ctx, q, token_out, basket_off, basket_token,
              basket_amount, limit_price, aoff, atok, o === nothing ? C_NULL : o, out) :
        ccall((:cfmm_quote_limit_orders, LIB), Cint, argq, ctx, q, token_out, basket_off, basket_token,
              basket_amount, limit_price, allowed, o === nothing ? C_NULL : o, out)
    GC.@preserve tok_off leg_off chk(ctx, quote_call(sizes))
    NT, L = tok_off[end], leg_off[end]
    paid, received, surplus, merit, status = zeros(max(NE, 1)), zeros(q), zeros(q), zeros(q), zeros(UInt8, q)
    sst, iters, fev = zeros(Cint, q), zeros(Cint, q), zeros(Cint, q)
    token, nu, psi = zeros(Int64, max(NT, 1)), zeros(max(NT, 1)), zeros(max(NT, 1))
    ltype, lpool, ld, ll = zeros(Cint, max(L, 1)), zeros(Int64, max(L, 1)), zeros(2, max(L, 1)), zeros(2, max(L, 1))
    GC.@preserve paid received surplus merit status sst iters fev tok_off token nu psi leg_off ltype lpool ld ll begin
        out = Ref(LimitOut(pointer(paid), pointer(received), pointer(status), pointer(sst), pointer(iters),
                           pointer(fev), pointer(merit), pointer(tok_off), NT, pointer(token), pointer(nu),
                           pointer(psi), pointer(leg_off), L, pointer(ltype), pointer(lpool), pointer(ld),
                           pointer(ll), pointer(surplus)))
        if execute && rows
            chk(ctx, ccall((:cfmm_execute_limit_orders_rows, LIB), Cint,
                (Ptr{Cvoid}, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{Int64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64},
                 Ptr{Int64}, Ptr{Int64}, Ptr{SubgraphOpts}, Ptr{LimitOut}),
                ctx, q, token_out, basket_off, basket_token, basket_amount, limit_price,
                min_received === nothing ? C_NULL : min_received, aoff, atok, o === nothing ? C_NULL : o, out))
        elseif execute
            chk(ctx, ccall((:cfmm_execute_limit_orders, LIB), Cint,
                (Ptr{Cvoid}, Int64, Ptr{Int64}, Ptr{Int64}, Ptr{Int64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64},
                 Ptr{UInt8}, Ptr{SubgraphOpts}, Ptr{LimitOut}),
                ctx, q, token_out, basket_off, basket_token, basket_amount, limit_price,
                min_received === nothing ? C_NULL : min_received, allowed, o === nothing ? C_NULL : o, out))
        else
            chk(ctx, quote_call(out))
        end
    end
    return (paid=paid[1:NE], received=received, surplus=surplus, status=status, solver_status=sst,
            iterations=iters, fun_evals=fev, merit=merit, tok_off=tok_off, token=token[1:NT], nu=nu[1:NT],
            psi=psi[1:NT], leg_off=leg_off, leg_type=ltype[1:L], leg_pool=lpool[1:L], leg_delta=ld[:, 1:L],
            leg_lambda=ll[:, 1:L])
end
quote_limit_orders(ctx, token_out, basket_off, basket_token, basket_amount, limit_price, allowed; opts=nothing) =
    _limit_orders(ctx, false, token_out, basket_off, basket_token, basket_amount, limit_price, allowed, nothing, opts)
execute_limit_orders!(ctx, token_out, basket_off, basket_token, basket_amount, limit_price, allowed;
                      min_received=nothing, opts=nothing) =
    _limit_orders(ctx, true, token_out, basket_off, basket_token, basket_amount, limit_price, allowed,
                  min_received, opts)

# UniV3 liquidity changes (cfmm_modify_univ3_liquidity / cfmm_get_univ3_ticks).  pools are 0-based
# UniV3 insertion indices; range is 2 x q (column j = (lo, hi) of row j).  univ3_ticks returns the
# current ladders of pools first .. first+count-1 in CSR form.  Like the rest of this file, never
# executed.
function modify_univ3_liquidity!(ctx, pools::Vector{Int64}, range::Matrix{Float64}, dL::Vector{Float64})
    size(range) == (2, length(pools)) == (2, length(dL)) ||
        throw(ArgumentError("range must be 2 x length(pools), dL of length(pools)"))
    chk(ctx, ccall((:cfmm_modify_univ3_liquidity, LIB), Cint,
        (Ptr{Cvoid}, Int64, Ptr{Int64}, Ptr{Float64}, Ptr{Float64}),
        ctx, length(pools), pools, range, dL))
end
function univ3_ticks(ctx, first::Integer, count::Integer)
    off = zeros(Int64, count + 1)
    chk(ctx, ccall((:cfmm_get_univ3_ticks, LIB), Cint,
        (Ptr{Cvoid}, Int64, Int64, Ptr{Int64}, Ptr{Float64}, Ptr{Float64}),
        ctx, first, count, off, C_NULL, C_NULL))
    lower, liq = zeros(Float64, off[end]), zeros(Float64, off[end])
    chk(ctx, ccall((:cfmm_get_univ3_ticks, LIB), Cint,
        (Ptr{Cvoid}, Int64, Int64, Ptr{Int64}, Ptr{Float64}, Ptr{Float64}),
        ctx, first, count, off, lower, liq))
    return off, lower, liq
end

end # module
