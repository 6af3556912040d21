# B200AdjointExt.jl -- Julia-side binding of libb200adj.so (include/b200adj.h).
#
# NOT EXECUTED IN THIS REPOSITORY'S ENVIRONMENT: Julia is not installed in the build image (SURVEY.md finding 6).
# The file is written against the same header the Python/ctypes host layer and the parity tests drive, and mirrors the
# extension precedent ext/SciMLSensitivityMooncakeExt.jl:123-240 of the reference: a new sensealg type plus a new
# method of SciMLBase._concrete_solve_adjoint returning (primal, pullback), and the ensemble entry the reference lacks
# (SURVEY.md 8b): an ensemble algorithm `EnsembleB200()` for `solve(::EnsembleProblem, alg, EnsembleB200(); ...)` with a
# ChainRules rrule on the batched solve (selected like DiffEqGPU.EnsembleGPUArray in docs/src/tutorials/data_parallel.md:293-302).
# What the device path does not support (B200ADJ_ERR_UNSUPPORTED, and the host-side checks below) is delegated to the wrapped
# reference sensealg; every OTHER error of the library is raised, never swallowed.
module B200AdjointExt

using SciMLSensitivity, SciMLBase
using SciMLSensitivity: BacksolveAdjoint, InterpolatingAdjoint, QuadratureAdjoint, GaussAdjoint, GaussKronrodAdjoint
using SciMLBase: ReturnCode
import ChainRulesCore
import ChainRulesCore: NoTangent

const libb200adj = get(ENV, "B200ADJ_LIB", "libb200adj.so")      # where the shared library lives (not a behaviour switch)

# ---- enums / cfg: field-for-field mirror of b200adj_cfg (176 bytes; checked against b200adj_sizeof_cfg) ----
@enum Family::Int32 FAM_LV = 0 FAM_LORENZ = 1 FAM_ROBERTSON = 2 FAM_SDE_LV = 3 FAM_MLP = 4 FAM_SDE_LINEAR = 5 FAM_BALL = 6 FAM_RELAX = 7
const SA_CODE = Dict(InterpolatingAdjoint => Int32(0), GaussAdjoint => Int32(1), QuadratureAdjoint => Int32(2),
    BacksolveAdjoint => Int32(3), GaussKronrodAdjoint => Int32(4))
const ST_TSIT5_FIXED, ST_ROSENBROCK23, ST_EM, ST_EULER_HEUN, ST_TSIT5_ADAPTIVE = Int32(0), Int32(1), Int32(2), Int32(3), Int32(4)
const COST_EXPLICIT, COST_AFFINE = Int32(0), Int32(1)
const FLAG_NO_START, FLAG_NO_CHECKPOINTING, FLAG_CKPT_EVERY_STEP = UInt32(1), UInt32(2), UInt32(4)
const ERR_UNSUPPORTED = Int32(-2)

"""
    B200PresetAffine(tstops, scale, shift; pscale = nothing, pshift = nothing)

The callback family the device path carries: at each `tstops[e]` the affect is `u .= scale[:, e] .* u .+ shift[:, e]` and,
optionally, `p .= pscale[:, e] .* p .+ pshift[:, e]` (`save_positions = (false, false)`; adaptive Tsit5, or fixed-step Tsit5
with the event times on the dt grid).  A plain marker object: passed as `callback =` to `solve(...; sensealg =
B200Adjoint(...))` it is consumed by the method below; for the reference path build the equivalent
`PresetTimeCallback(tstops, affect!)`.  `padd = (comp, param, coef)` (vectors of length E, 1-based indices, 0 = none) adds a
parameter to a state at event e, `u[comp[e]] += coef[e] * p[param[e]]` -- the "Dosing example" `integrator.u[1] += integrator.p[2]`
of test/Callbacks1/discrete_callbacks.jl:401-427 is `padd = ([1], [2], [1.0])` (adaptive Tsit5).
"""
struct B200PresetAffine
    tstops::Vector{Float64}; scale::Matrix{Float64}; shift::Matrix{Float64}
    pscale::Union{Nothing, Matrix{Float64}}; pshift::Union{Nothing, Matrix{Float64}}
    padd::Union{Nothing, Tuple{Vector{Int32}, Vector{Int32}, Vector{Float64}}}
end
B200PresetAffine(t, s, c; pscale = nothing, pshift = nothing, padd = nothing) =
    B200PresetAffine(collect(Float64, t), s, c, pscale, pshift,
                     padd === nothing ? nothing : (Int32.(padd[1]) .- Int32(1), max.(Int32.(padd[2]) .- Int32(1), Int32(0)), Float64.(padd[3])))

"""
    B200Crossing(idx, level = 0.0, direction = -1; scale = nothing, shift = nothing, pcomp = 0, pparam = 0, psign = 1.0, max_events = 64)

The state-dependent callback family of the device path: `ContinuousCallback(condition, affect!)` with
`condition(u, t, integrator) = u[idx] - level` (direction -1: `affect_neg!`-style downward crossings only, +1 upward, 0 both) and
`affect!`: `u .= scale .* u .+ shift`, then `u[pcomp] = psign * p[pparam] * u[pcomp]` when `pcomp > 0` (1-based here, 0-based at the
ABI).  The bouncing ball of docs/src/examples/hybrid_jump/bouncing_ball.md is `B200Crossing(1, 0.0, -1; pcomp = 2, pparam = 2,
psign = -1.0)`.  Adaptive Tsit5; every ensemble member finds its own event times on the device.
Parameter-dependent level and additive parameter affect (`lparam`, `lcoef`, `acomp`, `aparam`, `acoef`; 1-based, 0 = none):
`condition = u[1] - 3//4 * p[1]; affect! = u[1] += p[2]` of test/Callbacks2/continuous_callbacks.jl:317-345 is
`B200Crossing(1, 0.0, 0; lparam = 1, lcoef = 0.75, acomp = 1, aparam = 2, acoef = 1.0)`; the non-linear affect
`u[2] = u[2]^2` (:222-250) is `qcomp = 2` (`u[qcomp] = qcoef * u[qcomp]^2`).
"""
struct B200Crossing
    idx::Int; level::Float64; direction::Int
    scale::Union{Nothing, Vector{Float64}}; shift::Union{Nothing, Vector{Float64}}
    pcomp::Int; pparam::Int; psign::Float64; max_events::Int
    lparam::Int; lcoef::Float64; acomp::Int; aparam::Int; acoef::Float64; qcomp::Int; qcoef::Float64
end
B200Crossing(idx, level = 0.0, direction = -1; scale = nothing, shift = nothing, pcomp = 0, pparam = 0, psign = 1.0, max_events = 64,
             lparam = 0, lcoef = 0.0, acomp = 0, aparam = 0, acoef = 0.0, qcomp = 0, qcoef = 1.0) =
    B200Crossing(idx, level, direction, scale, shift, pcomp, pparam, psign, max_events, lparam, lcoef, acomp, aparam, acoef, qcomp, qcoef)

struct B200Cfg
    rhs_family::Int32; sensealg::Int32; stepper::Int32; dtype::Int32
    d::Int32; P::Int32; m::Int32; K::Int32
    N::Int64
    t0::Float64; t1::Float64; dt::Float64
    abstol::Float64; reltol::Float64
    quad_abstol::Float64; quad_reltol::Float64
    saveat::Ptr{Float64}
    shared_p::Int32; buffers_on_device::Int32; device::Int32; cost_kind::Int32
    cost_a::Float64; cost_b::Float64
    seed::UInt64; traj_offset::Int64
    checkpoint_every::Int32; flags::UInt32; mlp_hidden::Int32; block_threads::Int32
    max_steps::Int32; reserved0::Int32
end

function __init__()
    sz = ccall((:b200adj_sizeof_cfg, libb200adj), UInt32, ())
    sz == sizeof(B200Cfg) || error("b200adj_cfg layout mismatch: C $sz vs Julia $(sizeof(B200Cfg))")
end

"""
    B200Adjoint(inner; family, block_threads = 0, checkpoint_every = 1, devices = [0])

`sensealg = B200Adjoint(GaussAdjoint(); family = :lorenz)`: run the wrapped continuous adjoint on the B200 engine.
`family` names the hand-differentiated RHS family the problem's `f` belongs to (the role a user-supplied
`ODEFunction(f; vjp, vjp_p)` plays in src/derivative_wrappers.jl:284-359).  `devices`: CUDA ordinals the ensemble is sharded
over (one handle per device, members in contiguous blocks, dG/dp all-reduced inside `b200adj_reverse`).
"""
struct B200Adjoint{Inner} <: SciMLSensitivity.AbstractAdjointSensitivityAlgorithm{0, true, Val{:central}}
    inner::Inner
    family::Family
    block_threads::Int32
    checkpoint_every::Int32
    devices::Vector{Int32}
end
B200Adjoint(inner; family::Symbol, block_threads = 0, checkpoint_every = 1, devices = [0]) =
    B200Adjoint(inner, getfield(@__MODULE__, Symbol("FAM_", uppercase(String(family)))), Int32(block_threads),
        Int32(checkpoint_every), collect(Int32, devices))

"""
    EnsembleB200(; devices = [0])

Ensemble algorithm: `solve(EnsembleProblem(prob; prob_func), alg, EnsembleB200(); trajectories, saveat, sensealg =
B200Adjoint(...))` materialises `u0[d, N]` (and `p[P, N]` when `prob_func` changes `p`) on the host
(test/Core4/ensembles.jl:22-24) and runs ONE batched device solve; its rrule returns the batched pullback.
"""
struct EnsembleB200 <: SciMLBase.EnsembleAlgorithm
    devices::Vector{Int32}
end
EnsembleB200(; devices = [0]) = EnsembleB200(collect(Int32, devices))

struct B200Unsupported <: Exception
    msg::String
end
last_error(h) = unsafe_string(ccall((:b200adj_last_error, libb200adj), Cstring, (Ptr{Cvoid},), h))
# UNSUPPORTED -> a dedicated exception the entry points turn into delegation; everything else is an error
check(h, rc) = rc == 0 ? nothing : rc == ERR_UNSUPPORTED ? throw(B200Unsupported(last_error(h))) : error("b200adj error $rc: " * last_error(h))

const NOISE_NONE, NOISE_DIAGONAL, NOISE_GENERAL = Int32(0), Int32(1), Int32(2)
"""
    family_noise_kind(family) -> NOISE_NONE, NOISE_DIAGONAL or NOISE_GENERAL

The shape of a family's noise term (`b200adj_family_noise_kind`).  A general-noise SDE plug-in (`B200ADJ_FAMILY_SDE_GENERAL`,
G of size d x m) serves an `SDEProblem` with `noise_rate_prototype` of that size (scalar, non-diagonal or mixing noise);
EM + BacksolveAdjoint on it is UNSUPPORTED and so delegated to the wrapped sensealg.
"""
function family_noise_kind(family::Integer)
    k = Ref{Int32}(0)
    rc = ccall((:b200adj_family_noise_kind, libb200adj), Int32, (Int32, Ref{Int32}), Int32(family), k)
    rc == 0 || error("b200adj_family_noise_kind: unknown family id $family")
    return k[]
end

mutable struct Handle
    ptr::Ptr{Cvoid}
    function Handle(cfg::B200Cfg)
        ref = Ref{Ptr{Cvoid}}(C_NULL)
        rc = ccall((:b200adj_create, libb200adj), Int32, (Ref{B200Cfg}, Ref{Ptr{Cvoid}}), cfg, ref)
        rc == 0 || check(C_NULL, rc)
        h = new(ref[])
        finalizer(x -> ccall((:b200adj_destroy, libb200adj), Int32, (Ptr{Cvoid},), x.ptr), h)
        return h
    end
end

stepper_code(alg, adaptive) = nameof(typeof(alg)) === :Tsit5 ? (adaptive ? ST_TSIT5_ADAPTIVE : ST_TSIT5_FIXED) :
    nameof(typeof(alg)) === :EM ? ST_EM :
    nameof(typeof(alg)) === :EulerHeun ? ST_EULER_HEUN :
    nameof(typeof(alg)) === :Rosenbrock23 ? ST_ROSENBROCK23 : throw(B200Unsupported("solver $(typeof(alg))"))
is_sde_alg(alg) = nameof(typeof(alg)) in (:EM, :EulerHeun)

# One shard = one handle on one device.  Members [lo, hi) of the ensemble; buffers in the ABI's layouts.
struct Shard
    h::Handle; lo::Int; hi::Int
end

# ---- the batched solve + pullback on d x N / P (x N) arrays; `devices` shards the members ----
function b200_solve_adjoint(prob, alg, sensealg::B200Adjoint, U::AbstractMatrix{Float64}, p, originator, args...;
        save_start = true, save_end = true, saveat = Float64[], save_idxs = nothing, dt = nothing, callback = nothing,
        abstol = 1e-6, reltol = 1e-3, seed = UInt64(0), maxiters = 0, kwargs...)
    prob.f.mass_matrix === SciMLBase.I || throw(B200Unsupported("mass matrix"))
    p isa AbstractVecOrMat{Float64} || throw(B200Unsupported("parameters must be a flat Float64 vector or P x N matrix"))
    sde = is_sde_alg(alg)
    adaptive = !sde && get(kwargs, :adaptive, true)                  # OrdinaryDiffEq default; fixed step needs dt
    (adaptive || dt !== nothing) || throw(B200Unsupported("fixed-step solve without dt"))
    events = nothing; crossing = nothing
    if callback isa B200Crossing
        (nameof(typeof(alg)) === :Tsit5 && adaptive) || throw(B200Unsupported("state-dependent events: adaptive Tsit5"))
        crossing = callback
    elseif callback !== nothing
        (callback isa B200PresetAffine && nameof(typeof(alg)) === :Tsit5) || throw(B200Unsupported("callback outside the preset-time affine / crossing families"))
        events = callback
    end
    t0, t1 = prob.tspan
    # saveat::Number -> range with the end point appended; arrays sorted (concrete_solve.jl:718-725, 752-756); empty saveat =
    # every solver step is an output (:740-750) -- only the fixed-step grid is known before the solve
    ts = if saveat isa Number
        r = collect(t0:saveat:t1); r[end] == t1 || push!(r, t1); r
    elseif saveat isa AbstractArray && isempty(saveat)
        adaptive && throw(B200Unsupported("adaptive solve without saveat: the step sequence is per member"))
        collect(t0:dt:t1)
    else
        sort(collect(Float64, saveat))
    end
    # end points: dropped only for an EMPTY saveat (:740-750) and for Backsolve, whose forward solve keeps the solver's own
    # saving behaviour (:713-717); with a number or an array the output keeps t0 / t1 and `no_start` ignores the cotangent at t0
    if (saveat isa AbstractArray && isempty(saveat)) || sensealg.inner isa BacksolveAdjoint
        save_start || (!isempty(ts) && ts[1] == t0 && popfirst!(ts))
        save_end || (!isempty(ts) && ts[end] == t1 && pop!(ts))
    end
    no_start = !save_start && !isempty(ts) && ts[1] == t0                                    # concrete_solve.jl:962
    d, N = size(U)
    shared = p isa AbstractVector
    P = shared ? length(p) : size(p, 1)
    idxs = save_idxs === nothing ? collect(1:d) : save_idxs isa Number ? [save_idxs] : save_idxs === Colon() ? collect(1:d) : collect(save_idxs)
    K = length(ts)
    inner = sensealg.inner
    flags = (inner isa BacksolveAdjoint && !inner.checkpointing ? FLAG_NO_CHECKPOINTING : UInt32(0)) | (no_start ? FLAG_NO_START : UInt32(0))
    devs = sensealg.devices
    G = length(devs)
    bounds = [(g * N) ÷ G for g in 0:G]
    shards = Shard[]
    for g in 1:G
        lo, hi = bounds[g], bounds[g + 1]
        cfg = GC.@preserve ts B200Cfg(Int32(sensealg.family), SA_CODE[typeof(inner).name.wrapper], stepper_code(alg, adaptive), 0,
            d, P, sde ? d : 0, K, hi - lo, t0, t1, something(dt, 0.0), abstol, reltol,
            inner isa QuadratureAdjoint ? inner.abstol : 1e-6, inner isa QuadratureAdjoint ? inner.reltol : 1e-3,
            pointer(ts), shared, 0, devs[g], COST_EXPLICIT, 0.0, 0.0, seed, lo, sensealg.checkpoint_every, flags, 0,
            sensealg.block_threads, Int32(maxiters), 0)
        push!(shards, Shard(GC.@preserve(ts, Handle(cfg)), lo, hi))
    end
    if G > 1 && shared                                       # one communicator over the handles: b200adj_reverse all-reduces dp
        hp = [s.h.ptr for s in shards]
        check(hp[1], ccall((:b200adj_comm_init_all, libb200adj), Int32, (Ptr{Ptr{Cvoid}}, Int32), hp, G))
    end
    if events !== nothing        # [E], [E][d], [E][d], optional [E][P] x2 (row-major at the ABI = column-major transposed here)
        E = length(events.tstops)
        sc, sh = Matrix{Float64}(events.scale), Matrix{Float64}(events.shift)                 # d x E column-major = [E][d]
        psm = events.pscale === nothing ? nothing : Matrix{Float64}(events.pscale)
        pcm = events.pshift === nothing ? nothing : Matrix{Float64}(events.pshift)
        for s in shards
            GC.@preserve events sc sh psm pcm check(s.h.ptr, ccall((:b200adj_set_events, libb200adj), Int32,
                (Ptr{Cvoid}, Int32, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}),
                s.h.ptr, E, events.tstops, sc, sh, psm === nothing ? C_NULL : pointer(psm), pcm === nothing ? C_NULL : pointer(pcm)))
            if events.padd !== nothing
                pa = events.padd
                GC.@preserve pa check(s.h.ptr, ccall((:b200adj_set_event_param_shift, libb200adj), Int32,
                    (Ptr{Cvoid}, Ptr{Int32}, Ptr{Int32}, Ptr{Float64}), s.h.ptr, pa[1], pa[2], pa[3]))
            end
        end
    end
    if crossing !== nothing      # ContinuousCallback of the crossing family: each member finds its own event times in b200adj_forward
        c = crossing
        for s in shards
            GC.@preserve c check(s.h.ptr, ccall((:b200adj_set_continuous_callback, libb200adj), Int32,
                (Ptr{Cvoid}, Int32, Int32, Float64, Int32, Ptr{Float64}, Ptr{Float64}, Int32, Int32, Float64, Int32),
                s.h.ptr, 1, c.idx - 1, c.level, c.direction, c.scale === nothing ? C_NULL : pointer(c.scale),
                c.shift === nothing ? C_NULL : pointer(c.shift), c.pcomp - 1, max(c.pparam - 1, 0), c.psign, c.max_events))
            (c.lparam > 0 || c.acomp > 0 || c.qcomp > 0) && check(s.h.ptr, ccall((:b200adj_set_continuous_callback_params, libb200adj), Int32,
                (Ptr{Cvoid}, Int32, Float64, Int32, Int32, Float64, Int32, Float64),
                s.h.ptr, c.lparam - 1, c.lcoef, c.acomp - 1, max(c.aparam - 1, 0), c.acoef, c.qcomp - 1, c.qcoef))
        end
    end
    # forward: every shard on its own host thread (the calls block until the D2H copies are done)
    saved = [Array{Float64}(undef, s.hi - s.lo, d, K) for s in shards]                        # [K][d][n] in C order
    status = [Vector{Int32}(undef, s.hi - s.lo) for s in shards]
    U0s = [Matrix{Float64}(permutedims(U[:, (s.lo + 1):s.hi])) for s in shards]               # n x d column-major = [d][n]
    Ps = [shared ? Vector{Float64}(p) : Matrix{Float64}(permutedims(p[:, (s.lo + 1):s.hi])) for s in shards]
    Threads.@threads for g in 1:G
        s = shards[g]
        GC.@preserve U0s Ps saved status check(s.h.ptr, ccall((:b200adj_forward, libb200adj), Int32,
            (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Int32}), s.h.ptr, U0s[g], Ps[g], C_NULL, saved[g], status[g]))
    end
    u = [hcat((permutedims(saved[g][:, :, k])[idxs, :] for g in 1:G)...) for k in 1:K]         # length(idxs) x N per save time
    ok = all(all(==(0), st) for st in status)
    out = SciMLBase.build_solution(prob, alg, ts, u; retcode = ok ? ReturnCode.Success : ReturnCode.Unstable)

    function b200_adjoint_backpass(Δ)
        # Δ: Matrix (only_end), 3-array, VectorOfArray or Vector{Matrix} (concrete_solve.jl:777-868); rows = save_idxs, scattered
        # into a full-d jump with the other rows zero (:792-801)
        du0 = Matrix{Float64}(undef, d, N)
        dps = Vector{Any}(undef, G)
        Threads.@threads for g in 1:G
            s = shards[g]; n = s.hi - s.lo
            Δa = zeros(Float64, n, d, K)
            for k in 1:K
                Δk = Δ isa AbstractArray{<:Number, 3} ? view(Δ, :, :, k) : (K == 1 && Δ isa AbstractMatrix{<:Number}) ? Δ : Δ[k]
                Δa[:, idxs, k] .= permutedims(reshape(Δk, length(idxs), N)[:, (s.lo + 1):s.hi])
            end
            du0g = Matrix{Float64}(undef, n, d)
            dpg = shared ? Vector{Float64}(undef, P) : Matrix{Float64}(undef, n, P)
            GC.@preserve Δa du0g dpg check(s.h.ptr, ccall((:b200adj_reverse, libb200adj), Int32,
                (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}), s.h.ptr, Δa, du0g, dpg))
            du0[:, (s.lo + 1):s.hi] .= permutedims(du0g)
            dps[g] = dpg
        end
        dp = shared ? dps[1] : permutedims(vcat(dps...))                                      # shared: already summed over the shards
        return du0, dp
    end
    return out, b200_adjoint_backpass
end

# ---- the seam: SciMLBase._concrete_solve_adjoint(prob, alg, sensealg::B200Adjoint, u0, p, originator, args...; kw...) ----
# u0 is d x N (column i = member i) or a d-vector (N = 1); p a flat Vector (shared) or P x N matrix (per member).
function SciMLBase._concrete_solve_adjoint(
        prob::Union{SciMLBase.AbstractODEProblem, SciMLBase.AbstractSDEProblem},
        alg, sensealg::B200Adjoint, u0, p, originator::SciMLBase.ADOriginator, args...; kwargs...)
    delegate() = SciMLBase._concrete_solve_adjoint(prob, alg, sensealg.inner, u0, p, originator, args...; kwargs...)
    u0 isa AbstractVecOrMat{Float64} || return delegate()
    U = reshape(u0, size(u0, 1), :)
    local out, back
    try
        out, back = b200_solve_adjoint(prob, alg, sensealg, Matrix{Float64}(U), p, originator, args...; kwargs...)
    catch e
        e isa B200Unsupported || rethrow()                   # only "valid for the reference, not built here" falls back
        return delegate()
    end
    function pullback(Δ)
        du0, dp = back(ChainRulesCore.unthunk(Δ))
        du0_out = reshape(du0, size(u0))                     # concrete_solve.jl:978
        dp_out = p isa AbstractVector ? reshape(dp, size(p)) : dp                             # :980-986
        if originator isa SciMLBase.TrackerOriginator || originator isa SciMLBase.ReverseDiffOriginator
            (NoTangent(), NoTangent(), du0_out, dp_out, NoTangent(), ntuple(_ -> NoTangent(), length(args))...)
        else
            (NoTangent(), NoTangent(), NoTangent(), du0_out, dp_out, NoTangent(), ntuple(_ -> NoTangent(), length(args))...)
        end
    end
    return out, pullback
end

# ---- ensemble entry (absent in the reference, SURVEY.md finding 2): prob_func on the host, one batched device solve ----
function materialise(eprob::SciMLBase.EnsembleProblem, trajectories::Int)
    probs = [eprob.prob_func(eprob.prob, i, 1) for i in 1:trajectories]                      # test/Core4/ensembles.jl:22-24
    U = reduce(hcat, (vec(Float64.(q.u0)) for q in probs))
    same_p = all(q.p == probs[1].p for q in probs)
    p = same_p ? Vector{Float64}(vec(probs[1].p)) : reduce(hcat, (vec(Float64.(q.p)) for q in probs))
    return U, p
end

function SciMLBase.__solve(eprob::SciMLBase.EnsembleProblem, alg, ealg::EnsembleB200; trajectories, sensealg, kwargs...)
    sensealg isa B200Adjoint || error("EnsembleB200 needs sensealg = B200Adjoint(inner; family = ...)")
    U, p = materialise(eprob, trajectories)
    sa = B200Adjoint(sensealg.inner, sensealg.family, sensealg.block_threads, sensealg.checkpoint_every, ealg.devices)
    out, _ = b200_solve_adjoint(eprob.prob, alg, sa, U, p, SciMLBase.ChainRulesOriginator(); kwargs...)
    return out
end

function ChainRulesCore.rrule(::typeof(SciMLBase.__solve), eprob::SciMLBase.EnsembleProblem, alg, ealg::EnsembleB200; trajectories, sensealg, kwargs...)
    U, p = materialise(eprob, trajectories)
    sa = B200Adjoint(sensealg.inner, sensealg.family, sensealg.block_threads, sensealg.checkpoint_every, ealg.devices)
    out, back = b200_solve_adjoint(eprob.prob, alg, sa, U, p, SciMLBase.ChainRulesOriginator(); kwargs...)
    function ensemble_pullback(Δ)
        du0, dp = back(ChainRulesCore.unthunk(Δ))
        # the tangent of the EnsembleProblem: u0 / p of the base problem receive the member sums when prob_func leaves them alone
        dprob = ChainRulesCore.Tangent{typeof(eprob.prob)}(; u0 = reshape(sum(du0; dims = 2), size(eprob.prob.u0)), p = dp isa AbstractVector ? dp : vec(sum(dp; dims = 2)))
        return (NoTangent(), ChainRulesCore.Tangent{typeof(eprob)}(; prob = dprob), NoTangent(), NoTangent())
    end
    return out, ensemble_pullback
end

end # module
