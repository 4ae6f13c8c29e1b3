/*
 * cfmm_b200.h -- C ABI of libcfmm_b200.so: the H100-native replacement for the
 * dual-decomposition inner loop of CFMMRouter.jl (reference @ 5932e42).
 *
 * The reference has no FFI; the seam this ABI fills is INSIDE route!
 * (src/router.jl:58-108): the three call sites of find_arb!(r, v)
 * (router.jl:75, 93, 104, 107) and the two fold loops of the L-BFGS-B callback
 * (acc: router.jl:79-83, gradient scatter: router.jl:98-100).  One
 * cfmm_sweep() call = one find_arb!(r, v) over every pool + both folds.
 *
 * Conventions
 *  - extern "C", plain pointers and sizes, no C++/torch types.
 *  - every function returning int returns CFMM_OK (0) or a negative
 *    cfmm_status; nothing throws across the boundary.  The message for the
 *    last failure is cfmm_last_error(ctx) (ctx may be NULL for failures of
 *    cfmm_create).  Reference behaviour being replaced: Julia exceptions
 *    (ArgumentError from the ctors, src/cfmms.jl:77-78; BoundsError on a bad
 *    token index).
 *  - pointer arguments are caller-owned and borrowed for the duration of the
 *    call only; the context owns all device memory, streams and staging.
 *  - token indices are 1-BASED int64, exactly as Julia's cfmm.Ai
 *    (src/cfmms.jl:15, 87, 108); valid range 1..n_tokens, Ai[1] != Ai[2].
 *  - all values are IEEE fp64 (the only eltype the reference's tests use).
 *  - one context = one GPU = one shard of the pools.  A context is not
 *    thread-safe; use one per Router (the reference's callback is called
 *    synchronously from one thread, src/router.jl:105).
 *  - the library has NO CPU fallback: without a CUDA device every compute
 *    entry point fails with CFMM_ERR_CUDA.
 */
#ifndef CFMM_B200_H
#define CFMM_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct cfmm_ctx cfmm_ctx;

typedef enum cfmm_status {
  CFMM_OK = 0,
  CFMM_ERR_INVALID = -1, /* bad argument (ArgumentError / BoundsError analogue) */
  CFMM_ERR_CUDA = -2,    /* CUDA runtime failure or no device */
  CFMM_ERR_STATE = -3,   /* call order violated (e.g. sweep before finalize) */
  CFMM_ERR_NOMEM = -4,
  CFMM_ERR_COMM = -5     /* multi-GPU exchange set-up failure */
} cfmm_status;

typedef enum cfmm_pool_type {
  CFMM_POOL_PRODUCT = 0, /* ProductTwoCoin,       src/cfmms.jl:101-111 */
  CFMM_POOL_GEOMEAN = 1, /* GeometricMeanTwoCoin, src/cfmms.jl:152-165 */
  CFMM_POOL_UNIV3 = 2    /* UniV3,                src/cfmms.jl:226-245 */
} cfmm_pool_type;

/* ---- lifetime ------------------------------------------------------------ */

/* Replaces Router(objective, cfmms, n_tokens) (src/router.jl:18-35) for the
 * device-side state: creates an empty pool set on CUDA device `device`. */
int cfmm_create(cfmm_ctx **out, int device, int64_t n_tokens);
void cfmm_destroy(cfmm_ctx *ctx);
const char *cfmm_last_error(const cfmm_ctx *ctx);
/* "major.minor.patch" of the library */
const char *cfmm_version(void);

/* ---- pool ingest (before cfmm_finalize) ----------------------------------- */
/* Pools are numbered in GLOBAL INSERTION ORDER across all cfmm_add_* calls;
 * that is the order of r.cfmms / r.Δs / r.Λs on the reference side and the
 * order cfmm_get_trades returns. */

/* m x ProductTwoCoin(R, γ, idx) (src/cfmms.jl:101-111).
 * R: [2m] pool-major (R1,R2 per pool); gamma: [m]; Ai: [2m] 1-based. */
int cfmm_add_product(cfmm_ctx *ctx, int64_t m, const double *R,
                     const double *gamma, const int64_t *Ai);

/* m x GeometricMeanTwoCoin(R, w, γ, idx) (src/cfmms.jl:152-165). w: [2m]. */
int cfmm_add_geomean(cfmm_ctx *ctx, int64_t m, const double *R,
                     const double *gamma, const int64_t *Ai, const double *w);

/* m x UniV3(current_price, lower_ticks, liquidity, γ, Ai) (src/cfmms.jl:226-245)
 * in CSR form: pool i owns ticks tick_off[i] .. tick_off[i+1]-1 of
 * lower_ticks / liquidity (tick_off: [m+1], tick_off[0] == 0); lower_ticks
 * strictly decreasing within a pool.  current_tick is computed by the library
 * exactly as the reference ctor does (searchsortedlast rev=true, cfmms.jl:235);
 * a pool whose current_price exceeds its first lower tick (current_tick == 0,
 * a BoundsError in the reference) is rejected with CFMM_ERR_INVALID. */
int cfmm_add_univ3(cfmm_ctx *ctx, int64_t m, const double *current_price,
                   const double *gamma, const int64_t *Ai,
                   const int64_t *tick_off, const double *lower_ticks,
                   const double *liquidity);

/* Flat pool files: the ingest format for large pool sets (replaces building a
 * Vector{CFMM} of heap objects, src/router.jl:18-35, src/cfmms.jl:101-111).  Little-endian,
 * 64-byte header {"CFMMPOOL", u32 version 1, u32 cfmm_pool_type, i64 m, i64 n_tokens, pad},
 * then R [2m] f64, gamma [m] f64, Ai [2m] i64 (1-based), and w [2m] f64 for
 * GeometricMeanTwoCoin -- the arrays cfmm_add_product / cfmm_add_geomean take.
 * cfmm_add_pool_file mmaps the file and adds its pools (same validation, same errors). */
int cfmm_pool_file_write(const char *path, int type, int64_t n_tokens, int64_t m, const double *R,
                         const double *gamma, const int64_t *Ai, const double *w /* geomean */);
int cfmm_pool_file_info(const char *path, int *type, int64_t *n_tokens, int64_t *m);
int cfmm_add_pool_file(cfmm_ctx *ctx, const char *path);

/* Sort each pool type by its first token, lay it out SoA and upload. */
int cfmm_finalize(cfmm_ctx *ctx);

int64_t cfmm_num_pools(const cfmm_ctx *ctx);
int64_t cfmm_num_tokens(const cfmm_ctx *ctx);

/* ---- the hot path --------------------------------------------------------- */

/* One dual-gradient sweep at price vector v (host, [n_tokens]):
 *   find_arb!(r, v)                         src/router.jl:38-42
 *   acc  = Σ_i dot(Λ_i, v[Ai]) - dot(Δ_i, v[Ai])      src/router.jl:79-83
 *   psi  = Σ_i A_i (Λ_i - Δ_i)              src/router.jl:98-100 (G minus grad!(objective))
 * psi_out: host [n_tokens]; acc_out: host scalar.  With materialize != 0 the
 * per-pool trades Δ_i, Λ_i are also kept on the device (the final sweep of
 * route!, router.jl:107) for cfmm_get_trades.  Blocking: results are valid on
 * return.  When the context belongs to a multi-GPU group (cfmm_comm_attach),
 * psi/acc are the sums over all ranks' shards and every rank must call it.
 * Buffers from cfmm_host_alloc (pinned) avoid a staging copy; if acc_out ==
 * psi_out + n_tokens (one contiguous [psi ; acc] buffer) a single copy is used. */
int cfmm_sweep(cfmm_ctx *ctx, const double *v, double *psi_out,
               double *acc_out, int materialize);

/* Same sweep with ν already resident in device memory and the result left
 * there: d_v [n_tokens], d_psi_acc [n_tokens + 1] = [psi ; acc], both device
 * pointers on the context's device.  Enqueued on `stream` (a cudaStream_t;
 * NULL = the context's own stream) WITHOUT synchronising.  Stream rule: consecutive
 * operations of a context depend on each other (ping-pong accumulators, trade buffers,
 * reserves), so whenever an operation runs on a different stream than the previous one --
 * another caller stream, or the context's own stream, which cfmm_sweep, cfmm_get_trades,
 * cfmm_apply_trades, cfmm_update_reserves and cfmm_solve use -- the library makes the new
 * stream wait (event) for the work enqueued on the previous one.  The caller only has to
 * order its OWN reads of d_psi_acc after the sweep on `stream`. */
int cfmm_sweep_device(cfmm_ctx *ctx, const double *d_v, double *d_psi_acc,
                      int materialize, void *stream);

/* Zero-copy form: the result stays in a context-owned device buffer and
 * *d_psi_acc_out receives its address ([n_tokens + 1] fp64).  The buffer is
 * valid until the next sweep on this context is enqueued (two internal
 * accumulators alternate; each sweep clears the other one in-kernel, so no
 * memset or copy is launched). */
int cfmm_sweep_device_view(cfmm_ctx *ctx, const double *d_v, int materialize,
                           void *stream, const double **d_psi_acc_out);

/* Trades of the last materialising sweep, in global insertion order:
 * Delta, Lambda: host [2 * cfmm_num_pools] pool-major (r.Δs[i], r.Λs[i]). */
int cfmm_get_trades(cfmm_ctx *ctx, double *Delta, double *Lambda);

/* Overwrite reserves of pools [first, first+count) of one type, counted in
 * that type's own insertion order; R: [2*count].  (The reference reads
 * cfmm.R live on every sweep, so a caller that mutates reserves between
 * route! calls must push them.)  PRODUCT and GEOMEAN only. */
int cfmm_update_reserves(cfmm_ctx *ctx, int type, int64_t first, int64_t count,
                         const double *R);

/* Overwrite the state of UniV3 pools [first, first+count), counted in UniV3
 * insertion order.  current_price: [count], or NULL to keep the prices.
 * liquidity: the concatenated tick liquidities of those pools in their current
 * CSR order, or NULL to keep them.  The tick grid (lower_ticks, tick counts) is
 * the one of cfmm_add_univ3 / cfmm_append_univ3 until cfmm_modify_univ3_liquidity
 * inserts boundaries (cfmm_get_univ3_ticks reads the current one).  Prices are
 * validated as in cfmm_add_univ3 against the current first lower tick (a price
 * above the pool's first lower tick, or NaN, is rejected with CFMM_ERR_INVALID);
 * a rejected call changes no pool.  current_tick and every tick's BoundedProduct
 * (compute_at_tick, src/cfmms.jl:294-313) are recomputed on the device.
 * Synchronous. */
int cfmm_update_univ3(cfmm_ctx *ctx, int64_t first, int64_t count,
                      const double *current_price, const double *liquidity);

/* Apply the trades of the last materialising sweep to the device-resident pool
 * state (the update the reference intends with update_reserves!(r),
 * src/router.jl:127-132, whose per-CFMM method is defined nowhere).  Lets a
 * caller route repeatedly on evolving state without re-uploading pools.
 *
 * ProductTwoCoin / GeometricMeanTwoCoin: R <- R + γΔ − Λ (test/cfmms.jl:10).
 *
 * UniV3: the pool moves to the price its arbitrage walk (find_arb_pos,
 * src/cfmms.jl:321-337) trades it to.  With fee γ, current price q, first lower
 * tick T₁ = lower_ticks[1] and p = ν[a]/ν[b] at the ν of the last materialising
 * sweep (whichever entry point ran it; the library keeps a copy of that ν):
 *
 *   case (as src/cfmms.jl:347, 351)            new price q′
 *   γ·q <= p <= q/γ  (no trade)                q
 *   p < γ·q          (upper walk, :361)         min(p/γ, T₁)
 *   otherwise        (lower walk, :381)         min(γ·p, T₁)
 *   p/γ resp. γ·p is NaN or not > 0            q
 *
 * γ·q, q/γ, p/γ and γ·p are single IEEE operations, so q′ is bit-reproducible on
 * any host.  The clamp to T₁ covers a lower walk that drains tick 1 (no tick is
 * defined above T₁) and the case where p/γ rounds above q = T₁.  Then
 * current_tick′ = searchsortedlast(lower_ticks, q′, rev=true) (:235) and every
 * tick's BoundedProduct is compute_at_tick at (q′, current_tick′), recomputed on
 * the device for the pools whose price changed. */
int cfmm_apply_trades(cfmm_ctx *ctx);

/* ---- changing the pool set after cfmm_finalize ------------------------------------------
 * Pools are listed, drained and delisted while a caller routes block after block.  These
 * entry points change the set without a rebuild (cfmm_destroy, cfmm_add_*, cfmm_finalize).
 * Every change that alters the set (an append, a pool retired or restored, a compact) makes
 * cfmm_get_trades and cfmm_apply_trades return CFMM_ERR_STATE until the next materialising
 * sweep, and makes cfmm_sweep re-capture its graph.
 *
 * cfmm_append_*: the arguments and checks of the matching cfmm_add_*, valid only after
 * cfmm_finalize (before it: CFMM_ERR_STATE); a rejected call changes nothing.  The new pools take
 * the next global insertion indices (cfmm_num_pools grows) and the next indices of their type,
 * so cfmm_update_reserves, cfmm_update_univ3, cfmm_get_trades and the calls below address them
 * like ingested pools.  They live in a per-type tail, laid out like "tma_variant" -1 and swept
 * by the first-generation kernel after the type's main set; an append re-lays out only the tail
 * (from its current device state).  cfmm_compact folds the tails into the main layout. */
int cfmm_append_product(cfmm_ctx *ctx, int64_t m, const double *R,
                        const double *gamma, const int64_t *Ai);
int cfmm_append_geomean(cfmm_ctx *ctx, int64_t m, const double *R,
                        const double *gamma, const int64_t *Ai, const double *w);
int cfmm_append_univ3(cfmm_ctx *ctx, int64_t m, const double *current_price,
                      const double *gamma, const int64_t *Ai,
                      const int64_t *tick_off, const double *lower_ticks,
                      const double *liquidity);

/* Retire (active[j] == 0) or restore (active[j] != 0) the pools [first, first+count) of one
 * type, counted in that type's insertion order (appended pools included).  A retired pool
 * trades exactly zero and adds nothing to psi or acc; cfmm_apply_trades leaves it unchanged
 * (a UniV3 pool does not move).  Its state is kept: cfmm_update_reserves / cfmm_update_univ3
 * on a retired pool store the pushed state, which becomes live when it is restored.  Retiring
 * a retired pool or restoring an active one does nothing. */
int cfmm_set_active(cfmm_ctx *ctx, int type, int64_t first, int64_t count,
                    const uint8_t *active);

/* The current state of the pools [first, first+count) of one type, in that type's insertion
 * order: PRODUCT / GEOMEAN: the reserves, state [2*count] pool-major as cfmm_add_* takes them;
 * UNIV3: the current price, state [count].  Retired pools report the state they keep.
 * active (may be NULL): [count], 1 = active, 0 = retired. */
int cfmm_get_pool_state(cfmm_ctx *ctx, int type, int64_t first, int64_t count,
                        double *state, uint8_t *active);

/* Fold every type's appended pools into its main layout: the current state of all pools is
 * read back and laid out as cfmm_finalize does, with the same insertion indices (retired pools
 * stay retired), and the finalize calibration sweeps run again.  Afterwards a gradient sweep is
 * one launch per pool type again.  Costs about what cfmm_finalize costs. */
int cfmm_compact(cfmm_ctx *ctx);

/* ---- swaps against the device-resident pools ------------------------------------------
 * q swaps on pools of one type.  pool: [q] indices in that type's insertion order (appended
 * pools included).  tender: [2q] pool-major Δ, in the pool's ingest token order (Ai as given to
 * cfmm_add_*): each row (x, 0), (0, x) or (0, 0) with x finite and >= 0.  received: [2q] Λ,
 * nonzero only on the side opposite the tender.
 *
 * cfmm_quote_swaps prices every row against the current state on its own (rows on the same pool
 * do not see each other) and changes no state.  cfmm_execute_swaps applies the rows in batch
 * order: a row sees the effect of every earlier row on the same pool, and received holds what
 * each row actually got (the semantics of replaying a block).  Afterwards the state version
 * moves (captured sweep graphs see the new state), the guard-free range flag and the fixed-point
 * scale follow the new reserves, and the materialised trades (cfmm_get_trades) stay as they are.
 *
 * Both are synchronous.  Before cfmm_finalize they return CFMM_ERR_STATE; a bad type, an index
 * outside the type's pools, a NaN / Inf / negative tender or a row with both sides > 0 gives
 * CFMM_ERR_INVALID.  Every argument is checked before anything runs: a rejected call changes no
 * pool.  Retired pools (cfmm_set_active) receive (0, 0) and keep their state, parked or not.
 *
 * Trade rules, with δ = γ·x the tender net of the fee (forward_trade's γ*Δ[1], src/cfmms.jl:445),
 * for a tender of token 1 (token 2 is symmetric):
 *   ProductTwoCoin        λ₂ = min(R₂, R₂ − k/(R₁ + δ)), k = R₁·R₂: forward_amount of the
 *                         BoundedProduct (k, 0, 0, R₁, R₂) in the reference's operation order (bit
 *                         for bit; a tender below about eps·R₁ can give a λ a few ulp below zero,
 *                         as there).
 *   GeometricMeanTwoCoin  λ₂ = R₂·(1 − (R₁/(R₁ + δ))^η), η = w₁/w₂, clamped to [0, R₂]; evaluated as
 *                         −R₂·expm1(−η·log1p(δ/R₁)), within (4 + 2η)·eps·R₂ of the exact value.
 *   UniV3                 received = forward_trade(Δ, cfmm) (src/cfmms.jl:436-449), bit for bit: the
 *                         tick walk from the current tick through the upper ticks (token 1) or the
 *                         flipped lower ticks (token 2); empty ticks are walked through.
 * Execute, two-coin: R <- (R + γΔ) − Λ, the IEEE operations of cfmm_apply_trades.
 * Execute, UniV3: liquidity and ticks stay, the price moves to q′ (each step one IEEE operation):
 *   walk ended inside tick idx with δ′ left:  token 1: y = (R₁+α) + δ′, q′ = (k/y)/y
 *                                             token 2: y = (R₂+β) + δ′, q′ = (y/k)·y
 *                                             clamped to [lo(idx), hi(idx)], hi(idx) =
 *                                             lower_ticks[idx], lo(idx) = lower_ticks[idx+1] (0 for
 *                                             the last tick)
 *   walk exhausted every non-empty tick it reached: the far boundary of the last non-empty tick
 *                                             walked, lo(j) (token 1) or hi(j) (token 2)
 *   tender (0, 0), or no non-empty tick walked: unchanged
 *   then current_tick = searchsortedlast(lower_ticks, q′, rev=true) and the tick records are
 *   rebuilt as after cfmm_update_univ3. */
int cfmm_quote_swaps(cfmm_ctx *ctx, int type, int64_t q, const int64_t *pool,
                     const double *tender, double *received);
int cfmm_execute_swaps(cfmm_ctx *ctx, int type, int64_t q, const int64_t *pool,
                       const double *tender, double *received /* may be NULL */);

/* ---- exact-output swaps and slippage limits ----------------------------------------------
 * f(x) below is the exact-input quote of one pool at its current state as a function of the gross
 * tender x on one side: what cfmm_quote_swaps returns for that tender, bit for bit (f(0) = 0).
 *
 * Exact-output quote.  For a wanted output y > 0 on the side opposite the tender, the tender x* is
 * a crossing of f through y on the ordered doubles of [0, DBL_MAX]:
 *     f(x*) >= y, and x* = 0 or f(pred(x*)) < y        (pred: the next smaller double).
 * y = 0 gives x* = 0; x* = +inf when f(DBL_MAX) < y (unreachable) or the pool is retired.
 * The search is deterministic and bounded.  It starts from the estimate e (each step one IEEE
 * operation, round to nearest; log1p / expm1 are CUDA's), for a tender of the token with reserve
 * R_in and fee γ, wanting y of the other (R_out):
 *   ProductTwoCoin        e = ((R_in·R_out)/(R_out − y) − R_in)/γ, +inf if y >= R_out
 *   GeometricMeanTwoCoin  e = (R_in·expm1(−log1p(−(y/R_out))/η))/γ, η = w_in/w_out, +inf if y >= R_out
 *   UniV3                 the ticks of the forward walk in its order, each from compute_at_tick
 *                         with α, β, R_in, R_out flipped for a token-2 tender; s = 0, y′ = y:
 *                         a tick with y′ <= R_out ends the walk with
 *                           e = (s + (k/((R_out + β) − y′) − (R_in + α)))/γ,
 *                         any other tick does s = s + max_amount_pos, y′ = y′ − R_out; +inf if the
 *                         ticks run out.
 * Let o(x) be the bit pattern of a double x >= 0 read as an int64 (monotone in x), and
 * o_e = o(e) clamped to [1, o(DBL_MAX)] (1 for a NaN or e <= 0).  If f(e) >= y the search gallops
 * down: hi = o_e, then c = hi − 1, hi − 2, hi − 4, … (each step from the last c that still
 * reached y) until f(c) < y (lo = c) or c <= 0 (lo = 0).  Otherwise it gallops up: lo = o_e, then
 * c = lo + 1, lo + 2, lo + 4, … capped at o(DBL_MAX), until f(c) >= y (hi = c); unreachable
 * when o(DBL_MAX) falls short.  It then bisects, mid = lo + (hi − lo)/2, keeping f(lo) < y <=
 * f(hi), until hi = lo + 1, and x* = hi.  At most 1 + 63 + 62 evaluations of f.
 *   ProductTwoCoin: f is non-decreasing in x.  γ·x, R_in + δ, k/·, R_out − · and min(R_out, ·)
 *   are each correctly rounded monotone functions (non-decreasing, or non-increasing for k/·
 *   with the subtraction reversing it), so their composition is monotone; the crossing is unique
 *   and x* is the least double that receives at least y.
 *   UniV3 and GeometricMeanTwoCoin: f can step back by a few ulp (where a UniV3 walk enters a new
 *   tick, whose first output can round slightly below zero; through CUDA's log1p and expm1), so
 *   several crossings can lie within a few ulp.  x* is the one this search finds.
 *
 * cfmm_quote_swaps_exact_out: want [2q] pool-major, (0, y) receives token 2 for a tender of token
 * 1 and (y, 0) the reverse (ingest token order, as cfmm_quote_swaps); tender [2q] gets (x*, 0) or
 * (0, x*).  Rows are priced on the current state on their own; no state changes.
 *
 * cfmm_execute_swap_orders: rows of kind CFMM_SWAP_EXACT_IN (amount = the tender, as
 * cfmm_execute_swaps; limit = the minimum received, NULL means 0) or CFMM_SWAP_EXACT_OUT (amount =
 * the wanted output, as above; limit = the maximum tender, NULL or +inf means none), applied in
 * batch order per pool.  An exact-out row's x* is computed against the pool's state after the
 * earlier rows of the batch.  A row reverts, changing nothing, when its pool is retired
 * (CFMM_ORDER_RETIRED), an exact-in row receives less than its limit or an exact-out row's x*
 * exceeds its limit (CFMM_ORDER_LIMIT), or y is unreachable (CFMM_ORDER_UNREACHABLE); later rows
 * see the state without it.  An equal limit fills.  A filled row (CFMM_ORDER_FILLED) runs the
 * transition of cfmm_execute_swaps with its tender, so the filled rows of a batch leave exactly
 * the state, and receive exactly what, cfmm_execute_swaps with their paid tenders gives.  Per row:
 * paid [2q] the gross tender on the tender side, received [2q] (an exact-out row receives f(x*) >=
 * y), status [q]; a reverted row pays and receives (0, 0).  The bookkeeping afterwards is that of
 * cfmm_execute_swaps.
 *
 * Both are synchronous.  Before cfmm_finalize: CFMM_ERR_STATE.  CFMM_ERR_INVALID before anything
 * runs, so no pool changes, for a bad type, a pool outside the type's pools, a kind other than 0
 * or 1, an amount that is NaN, Inf, negative or has both sides > 0, a limit that is NaN or
 * negative, or a limit of +inf on an exact-in row.  q == 0 does nothing. */
#define CFMM_SWAP_EXACT_IN 0
#define CFMM_SWAP_EXACT_OUT 1
#define CFMM_ORDER_FILLED 0
#define CFMM_ORDER_LIMIT 1
#define CFMM_ORDER_UNREACHABLE 2
#define CFMM_ORDER_RETIRED 3
int cfmm_quote_swaps_exact_out(cfmm_ctx *ctx, int type, int64_t q, const int64_t *pool,
                               const double *want /* [2q] */, double *tender /* [2q], +inf unreachable */);
int cfmm_execute_swap_orders(cfmm_ctx *ctx, int type, int64_t q, const int64_t *pool,
                             const uint8_t *kind /* [q] */, const double *amount /* [2q] */,
                             const double *limit /* [q] or NULL */, double *paid /* [2q] or NULL */,
                             double *received /* [2q] or NULL */, uint8_t *status /* [q] or NULL */);

/* ---- multi-hop swap paths ----------------------------------------------------------------
 * A path tenders token t₀ to its first pool, tenders what that pool pays out to the next, and so
 * on; one limit covers the whole path, and a path whose limit fails reverts every hop.  Path j is
 * the hops hop_off[j] .. hop_off[j+1]) (hop_off [q+1], hop_off[0] = 0, 1..CFMM_PATH_MAX_HOPS hops
 * per path; H = hop_off[q]).  Hop h is pool hop_pool[h] of type hop_type[h], addressed as
 * cfmm_quote_swaps addresses a pool (the type's insertion order, appended pools included).  The
 * pools of one path are distinct, so its hops never see each other.
 *
 * Tokens.  t₀ = token_in[j] (1-based).  Hop h's pool must hold t_{h−1}, and t_h is its other token.
 * The hop tenders token 1 of the pool's ingest order (Ai as given to cfmm_add_* / cfmm_append_*)
 * when t_{h−1} is that token, token 2 otherwise.
 *
 * f_h(x) is the exact-input quote of hop h's pool at its state before the path: what
 * cfmm_quote_swaps returns for that tender, bit for bit (f_h(0) = 0).
 *   Exact-in (kind CFMM_SWAP_EXACT_IN).  x₁ = amount; λ_h = f_h(x_h); x_{h+1} = λ_h if λ_h > 0,
 *     else 0 (a ProductTwoCoin output can be a few ulp below zero, see the swaps section: it is
 *     passed on as 0, the reported λ_h keeps its value).  The limit is the minimum λ_n (NULL: 0).
 *   Exact-out (kind CFMM_SWAP_EXACT_OUT).  y_n = amount; for h = n … 1, x_h is the crossing of f_h
 *     through y_h found by the search of cfmm_quote_swaps_exact_out, bit for bit (0 for y_h = 0), and
 *     y_{h−1} = x_h.  λ_h = f_h(x_h) >= y_h: the surplus λ_h − x_{h+1} >= 0 stays with the trader.
 *     The limit is the maximum x₁ (NULL or +inf: none).
 * Status (CFMM_ORDER_*), first match: RETIRED when a hop's pool is retired; UNREACHABLE when some
 * x_h = +inf; LIMIT (execute only) when λ_n < limit (exact-in) or x₁ > limit (exact-out), so an
 * equal limit fills; otherwise FILLED.  A path that does not fill reports 0 as every hop's tender
 * and received.  Per hop, hop_tender [H] = x_h (gross, in the tendered token) and hop_received
 * [H] = λ_h; the path paid hop_tender[hop_off[j]] and received hop_received[hop_off[j+1] − 1].
 *
 * cfmm_quote_paths prices every path on the current state on its own; no state changes.
 * cfmm_execute_paths runs the paths in batch order: path j is priced on the state every earlier
 * filled path left, and a filled path runs the transition of cfmm_execute_swaps on each hop with
 * tender x_h.  So the final state and every hop amount are bit-identical to running, path by path,
 * each hop of each filled path as a one-row cfmm_execute_swaps call with that tender.  A reverted
 * path changes nothing.  Afterwards every set a filled path touched gets the bookkeeping of
 * cfmm_execute_swaps (state version, guard-free range flag, fixed-point scale, UniV3 tick records);
 * the materialised trades stay.  Paths that share no pool run in parallel: path j's level is 1 +
 * the largest level of an earlier path sharing one of its pools, and each level is one launch.
 *
 * Both are synchronous.  Before cfmm_finalize: CFMM_ERR_STATE.  q == 0 does nothing.
 * CFMM_ERR_INVALID, before anything changes, for: q < 0 or a null array; hop_off not starting at 0,
 * decreasing, or a path of 0 or more than CFMM_PATH_MAX_HOPS hops; a bad type or a pool outside the
 * type's pools; the same pool twice in one path; token_in outside 1..n_tokens; a hop whose pool
 * does not hold the token that reaches it (the message names the first such path and hop); a kind
 * other than 0 or 1; an amount that is NaN, Inf or negative; a limit that is NaN or negative, or
 * +inf on an exact-in path. */
#define CFMM_PATH_MAX_HOPS 8
int cfmm_quote_paths(cfmm_ctx *ctx, int64_t q, const int64_t *hop_off /* [q+1] */,
                     const int *hop_type /* [H] */, const int64_t *hop_pool /* [H] */,
                     const int64_t *token_in /* [q], 1-based */, const uint8_t *kind /* [q] */,
                     const double *amount /* [q] */, double *hop_tender /* [H] */,
                     double *hop_received /* [H] */, uint8_t *status /* [q] */);
int cfmm_execute_paths(cfmm_ctx *ctx, int64_t q, const int64_t *hop_off, const int *hop_type,
                       const int64_t *hop_pool, const int64_t *token_in, const uint8_t *kind,
                       const double *amount, const double *limit /* [q] or NULL */,
                       double *hop_tender /* [H] or NULL */, double *hop_received /* [H] or NULL */,
                       uint8_t *status /* [q] or NULL */);

/* ---- the pools of a token pair -----------------------------------------------------------
 * For each row, the pools that hold the unordered token pair {token_a[j], token_b[j]} (1-based,
 * distinct): all three types, main sets and appended pools, in global insertion order (the
 * cfmm_num_pools numbering).  count [q] is always written.  When cap >= Σ count, the rows' lists
 * follow one another in row order: type_out [Σ count] (cfmm_pool_type), pool_out [Σ count] (the
 * index in the type's insertion order, as cfmm_quote_swaps addresses a pool) and active_out
 * [Σ count] (0 = retired); any of them may be NULL.  So a first call with cap = 0 sizes the
 * outputs.  The index behind it is built on the device on the first call that needs it after
 * cfmm_finalize, cfmm_append_* or cfmm_compact (a key min(a,b)·n_tokens + max(a,b) per pool, a
 * stable radix sort, a run-length pass; lookups bisect the distinct keys) and kept; retiring or
 * restoring a pool does not rebuild it.  Synchronous.  Before cfmm_finalize: CFMM_ERR_STATE;
 * tokens outside 1..n_tokens or equal, q < 0 or a null token / count array: CFMM_ERR_INVALID. */
int cfmm_pair_pools(cfmm_ctx *ctx, int64_t q, const int64_t *token_a /* [q] */,
                    const int64_t *token_b /* [q] */, int64_t *count /* [q] */, int64_t cap,
                    int *type_out, int64_t *pool_out, uint8_t *active_out);

/* ---- orders split optimally across every pool of their token pair ------------------------
 * A row sells token j = token_in[r] for token i = token_out[r] (1-based, distinct) over every pool
 * that holds {i, j} (cfmm_pair_pools order).  This is route! with Swap(i, j, δ, 2) over those pools
 * only (src/objectives.jl:92-146, src/router.jl:58-108): with ν_i = 1 its dual has one variable,
 * s = ν_j/ν_i, and the optimal split is the pools' response at the s* where their net intake of j
 * matches the order (dual decomposition, docs/src/method.md).
 *
 * Pool response at s.  ν[i] = 1.0, ν[j] = s.  Pool k's legs (Δ_k, Λ_k) are the materialising
 * find_arb! at ν[Ai] (src/cfmms.jl:125-140 ProductTwoCoin, :180-196 GeometricMeanTwoCoin,
 * :339-395 UniV3, the UniV3 walk from the pool's current price and ladder): what cfmm_sweep with
 * materialize = 1 reads back through cfmm_get_trades, bit for bit.  Retired pools give (0, 0).
 * Legs are in the pool's ingest token order (a ProductTwoCoin pool stored with its tokens exchanged
 * is mapped back).
 *
 * Sums.  N(s) = Σ_k (Δ_j,k − Λ_j,k), the pools' net intake of j, non-increasing in s, and
 * O(s) = Σ_k (Λ_i,k − Δ_i,k), their output of i; each term one IEEE subtraction.  k runs over the
 * pair's pools in order, and the sum has one fixed shape: partial l (l = 0 … 31) adds the terms
 * k ≡ l (mod 32) in increasing k, starting from +0.0; then for m = 16, 8, 4, 2, 1 every partial
 * becomes p_l + p_(l xor m).  The result is p_0 (every p_l ends equal).  No atomics.
 *
 * Search, on o(s), the bit pattern of s > 0 read as an int64, over [o(DBL_MIN), o(DBL_MAX)].
 * enough(s) is N(s) > δ (a NaN counts as true) for exact-in (kind CFMM_SWAP_EXACT_IN, amount δ
 * tendered), O(s) >= y for exact-out (CFMM_SWAP_EXACT_OUT, amount y wanted); true at small s.
 *   start   e = the largest no-trade boundary over the pair's active pools (NaNs ignored), the s
 *           below which pool k starts to take j, each step one IEEE operation:
 *             ProductTwoCoin        (γ·R_i)/R_j
 *             GeometricMeanTwoCoin  ((γ·w_j)·R_i)/(w_i·R_j)
 *             UniV3                 γ·q when its token 1 is j, γ/q when it is i (q: current price)
 *           o_e = o(e) clamped to [o(DBL_MIN), o(DBL_MAX)] (o(DBL_MIN) when e is NaN or < DBL_MIN).
 *   gallop  if enough(o_e): lo = o_e, then c = lo + 1, lo + 2, lo + 4, … capped at o(DBL_MAX),
 *           lo = c while enough(c), until !enough(c) (hi = c); unreachable when lo = o(DBL_MAX).
 *           Otherwise hi = o_e, then c = hi − 1, hi − 2, hi − 4, … capped at o(DBL_MIN), hi = c
 *           while !enough(c), until enough(c) (lo = c); unreachable when hi = o(DBL_MIN).
 *   bisect  mid = lo + (hi − lo)/2 replaces lo (enough) or hi (not) until hi = lo + 1.
 *   result  s* = hi for exact-in (N(s*) <= δ), s* = lo for exact-out (O(s*) >= y).
 * Every row costs at most 1 + 63 + 62 evaluations of the pair's pools in the search and one more at
 * s*, which writes the legs: 127.  A row with amount 0 fills with zeros and runs no search (the
 * split never hands out free arbitrage to an empty order).  A pair no active pool holds, and a
 * gallop that reaches either end without a bracket (the pools cannot absorb δ, or cannot deliver
 * y, e.g. a UniV3 pool whose last tick is empty), give CFMM_ORDER_UNREACHABLE.
 *
 * What a fill means.  paid = N(s*) of j, received = O(s*) of i, price = s* (0 for an unreachable
 * row or amount 0), and each pool trades its legs at s*.  When the pair's pools disagree on the
 * price by more than their fees, the optimal split also arbitrages between them, as route! would:
 * some legs then pay out j or take in i, and the legs show it.
 *
 * cfmm_quote_split_orders prices every row on the current state on its own; no state changes.
 * cfmm_execute_split_orders runs the rows in batch order, each priced on the state the earlier
 * filled rows left.  limit (NULL: none) is the minimum received for exact-in and the maximum paid
 * for exact-out; a row whose limit fails reverts with CFMM_ORDER_LIMIT (its price is still
 * reported), and an equal limit fills.  A filled row applies to each of its pair's active pools the
 * transition of cfmm_apply_trades at its ν: two-coin R <- (R + γΔ) − Λ; UniV3 the q′ rule there
 * with p = ν[a]/ν[b] (current tick updated with it).  Rows of one pair run in order in one warp;
 * pairs share no pool and run in parallel.  Afterwards the bookkeeping of cfmm_execute_swaps
 * (state version, guard-free range flag, fixed-point scale, UniV3 tick records); the materialised
 * trades stay.  Reverted and unreachable rows change nothing and pay and receive 0.
 *
 * Per row: paid, received, price [q], status [q] (CFMM_ORDER_*); legs (optional): leg_delta,
 * leg_lambda [2L], L = the sum of the rows' pool counts (cfmm_pair_pools), row after row, each
 * pool's (Δ, Λ) pool-major in the pair's order as cfmm_get_trades lays them out; 0 for a row that
 * does not fill.  Every output may be NULL.
 *
 * Both are synchronous.  Before cfmm_finalize: CFMM_ERR_STATE.  q == 0 does nothing.
 * CFMM_ERR_INVALID before anything changes for: q < 0 or a null input array; tokens outside
 * 1..n_tokens or token_in == token_out; a kind other than 0 or 1; an amount that is NaN, Inf or
 * negative; a limit that is NaN or negative, or +inf on an exact-in row. */
int cfmm_quote_split_orders(cfmm_ctx *ctx, int64_t q, const int64_t *token_in /* [q] */,
                            const int64_t *token_out /* [q] */, const uint8_t *kind /* [q] */,
                            const double *amount /* [q] */, double *paid /* [q] */,
                            double *received /* [q] */, double *price /* [q] */,
                            uint8_t *status /* [q] */, double *leg_delta /* [2L] or NULL */,
                            double *leg_lambda /* [2L] or NULL */);
int cfmm_execute_split_orders(cfmm_ctx *ctx, int64_t q, const int64_t *token_in,
                              const int64_t *token_out, const uint8_t *kind, const double *amount,
                              const double *limit /* [q] or NULL */, double *paid, double *received,
                              double *price, uint8_t *status, double *leg_delta,
                              double *leg_lambda);

/* ---- orders routed over their pair and two-hop routes through hub tokens -----------------
 * A row sells j = token_in[r] for i = token_out[r] (1-based, distinct) over the pools of {j, i}
 * (the direct pools) and, for each of its hubs h = hubs[hub_off[r] .. hub_off[r+1]) (1-based,
 * 0..CFMM_ROUTE_MAX_HUBS per row, distinct, neither i nor j), the pools of {j, h} and of {h, i}
 * (hub h's pools), each list in cfmm_pair_pools order.  Pools between two hubs are not used.  This
 * is route! with Swap(i, j, δ) over exactly these pools (src/objectives.jl:92-146,
 * docs/src/method.md).  With ν_i = 1, ν_j = s and ν_h = t_h, hub h's price only enters hub h's pools,
 * so the dual separates: for each s, t_h solves "hub h's pools net to zero in h" (monotone in t_h),
 * and what is left is the split's convex problem in s, whose slope is δ − N(s).  General pool
 * graphs, with pools between hubs, remain cfmm_solve's.
 *
 * Pool response at (s, t).  A pool's legs are split orders' (the materialising find_arb! at ν[Ai],
 * mapped back to the ingest token order; retired pools give (0, 0)) at ν_i = 1, ν_j = s, ν_h = t_h.
 *
 * Sums, each with split orders' warp tree over one list of pools (partial l adds the terms of
 * pools k ≡ l (mod 32) in increasing k from +0.0, then the xor butterfly 16 … 1):
 *   direct    over the direct pools: N_d = Σ (Δ_j − Λ_j), O_d = Σ (Λ_i − Δ_i), split orders' bits;
 *   hub h     over its {j, h} pools followed by its {h, i} pools: N_h = Σ (Δ_j − Λ_j),
 *             O_h = Σ (Λ_i − Δ_i) and H_h = Σ (Λ_h − Δ_h), a pool adding nothing to a sum whose
 *             token it does not hold (each term one IEEE subtraction);
 *   N(s) = ((N_d + N_h₁) + N_h₂) + … and O(s) likewise, in the row's hub order, each hub's sums
 *   taken at its t_h(s).  With no hubs, or hubs that hold no pools, N and O are split orders'.
 *
 * Search.  Both searches are split orders' gallop and bisection on the ordinals o(x) of the doubles
 * in [DBL_MIN, DBL_MAX], from a start o(e) clamped to that range (o(DBL_MIN) for a NaN e):
 *   inner (hub h, at one s)  enough(t) is !(H_h(t) >= 0) (a NaN counts as true).  t_h(s) = hi, the
 *           smallest ordinal the search finds with H_h >= 0, so the hub surplus is never negative;
 *           when H_h(DBL_MIN) >= 0 already (the gallop down reaches o(DBL_MIN)), t_h = DBL_MIN.
 *           The first inner search of a row starts from the largest no-trade boundary of the hub's
 *           active {h, i} pools (split orders' boundary with h in j's role); every later one starts
 *           from the t_h the row's previous outer evaluation found.  H_h < 0 at t = DBL_MAX (the
 *           gallop up reaches o(DBL_MAX)) makes the row CFMM_ORDER_UNREACHABLE.
 *   outer   split orders' search on s with their enough (exact-in N(s) > δ, exact-out O(s) >= y),
 *           each evaluation running every hub's inner search.  Its start e is the largest of the
 *           direct pools' boundaries (split orders') and, for each hub with an active pool on both
 *           sides, b_jh · b_hi (one IEEE multiply; b_jh the largest boundary of its active {j, h}
 *           pools with j in j's role, b_hi that of its {h, i} pools with h in j's role).
 *           s* = hi for exact-in, lo for exact-out; t_h* = the t_h found at s* by that evaluation.
 * The legs pass at s* reuses t_h* and runs no inner search.  So a row costs at most 127 evaluations
 * of the direct pools and, for each hub, 126·126 + 1 of its pools.  A row with no hubs is split
 * orders' row bit for bit (legs, status and price included).  A row none of whose pools is active
 * is UNREACHABLE, and amount 0 fills with zeros and runs no search.
 *
 * Outputs, each optional (NULL): paid = N(s*), received = O(s*), price = s* (0 when unreachable or
 * amount 0), status [q] (CFMM_ORDER_*); hub_price [Σ] = t_h* (0 when price is 0); hub_surplus [Σ]
 * = H_h(t_h*) >= 0, the hub token left with the trader (0 unless filled); legs leg_delta,
 * leg_lambda [2L], row after row, each row's lists concatenated in the order {j, i}, {j, h₁},
 * {h₁, i}, {j, h₂}, …, so that one cfmm_pair_pools call on those pairs identifies them; 0 for a row
 * that does not fill.
 *
 * cfmm_quote_routed_orders prices every row on the current state on its own; no state changes.
 * cfmm_execute_routed_orders runs the rows in batch order with split orders' limits and revert rule.
 * A filled row applies cfmm_apply_trades' transition at its ν to each of its active pools (two-coin
 * R <- (R + γΔ) − Λ; UniV3 the q′ rule with p = ν[a]/ν[b], current tick updated).  Two rows
 * conflict when they share a token pair (a pool belongs to one pair): a row's level is 1 + the
 * highest level of an earlier row sharing one of its pairs, and each level is one launch of one CTA
 * per row (warp 0 the direct pools, warp 1 + h hub h).  Afterwards the bookkeeping of
 * cfmm_execute_swaps.  Reverted and unreachable rows change nothing.
 *
 * Both are synchronous.  Before cfmm_finalize: CFMM_ERR_STATE.  q == 0 does nothing.
 * CFMM_ERR_INVALID before anything changes for every argument split orders reject, and for: a null
 * hub_off, hub_off[0] != 0, a row with fewer than 0 or more than CFMM_ROUTE_MAX_HUBS hubs, a null
 * hubs with hub_off[q] > 0, a hub outside 1..n_tokens, equal to the row's i or j, or listed twice in
 * the row. */
#define CFMM_ROUTE_MAX_HUBS 7
int cfmm_quote_routed_orders(cfmm_ctx *ctx, int64_t q, const int64_t *token_in /* [q] */,
                             const int64_t *token_out /* [q] */, const uint8_t *kind /* [q] */,
                             const double *amount /* [q] */, const int64_t *hub_off /* [q+1] */,
                             const int64_t *hubs /* [Σ] */, double *paid /* [q] */,
                             double *received /* [q] */, double *price /* [q] */,
                             uint8_t *status /* [q] */, double *hub_price /* [Σ] */,
                             double *hub_surplus /* [Σ] */, double *leg_delta /* [2L] */,
                             double *leg_lambda /* [2L] */);
int cfmm_execute_routed_orders(cfmm_ctx *ctx, int64_t q, const int64_t *token_in,
                               const int64_t *token_out, const uint8_t *kind, const double *amount,
                               const double *limit /* [q] or NULL */, const int64_t *hub_off,
                               const int64_t *hubs, double *paid, double *received, double *price,
                               uint8_t *status, double *hub_price, double *hub_surplus,
                               double *leg_delta, double *leg_lambda);

/* ---- arbitrage: pair cycles and triangles through base tokens --------------------------------
 * An arbitrage row names a base token p = base[r] (the profit token), another token x = other[r]
 * (1-based, distinct) and hubs y = hubs[hub_off[r] .. hub_off[r+1]) with routed rows' rules (at most
 * CFMM_ROUTE_MAX_HUBS, distinct, neither p nor x).  Its pools are those of {x, p}, {x, y} and {y, p}:
 * the pair cycle p → x → p and one triangle p → x → y → p (either direction) per hub.  The row is
 * route! with BasketLiquidation(p, 0) over these pools: maximise the output of p while x and every y
 * end non-negative.  That is the routed exact-in row j = x, i = p with δ = 0, and its dual separates
 * in the same way, so the row runs routed rows' searches (start, gallop, bisection, inner hub
 * searches, sums and their order, UNREACHABLE rules) with enough(s) = N(s) > 0 (a NaN counts as
 * true) and s* = hi.  It runs the search where a routed row with amount 0 does not, and a row whose
 * pair {x, p} no pool holds is CFMM_ORDER_UNREACHABLE.
 *
 * Outputs, each optional (NULL), per row: profit = O(s*), the p the cycle yields; surplus_in =
 * 0.0 − N(s*) >= 0 (one IEEE subtraction), the x left with the trader; price = s* (0 when
 * unreachable); status; hub_price [Σ] = t_h*, hub_surplus [Σ] = H_h(t_h*) >= 0; legs leg_delta,
 * leg_lambda [2L] in routed rows' list order ({x, p}, {x, y₁}, {y₁, p}, …).  Rows that do not fill
 * report 0 for profit, surplus and the legs.  With no arbitrage left, the row fills with profit 0.
 * By weak duality O >= s·N − Σ t_h·H_h, so rounding can leave a filled profit a few ulps below 0.
 *
 * cfmm_quote_arbitrage prices every row on the current state on its own; no state changes.
 * cfmm_execute_arbitrage runs the rows in batch order, each on the state the earlier filled rows
 * left, with routed rows' levels, transitions and bookkeeping.  min_profit [q] (NULL: 0) is each
 * row's limit: a row with profit < min_profit reverts with CFMM_ORDER_LIMIT (an equal value fills).
 *
 * cfmm_scan_arbitrage finds the rows worth running for distinct base tokens base[nb], each with
 * min_profit[b] (finite, > 0, in units of that base token), with up to max_hubs (0..7) hubs per row.
 * It changes no state and is synchronous.  Its steps:
 *   adjacency  for every distinct token pair {a, b} of the pools (retired included), the entries
 *            a → b and b → a sorted by (token, neighbour); built on the device with the pair index
 *            (first use after cfmm_finalize, cfmm_append_* or cfmm_compact; kept across retire and
 *            restore).  2·n_pairs entries of 8 bytes.
 *   rates    r(a → b) = the largest, over the active pools of {a, b}, of the start boundary of
 *            routed rows with a in j's role (ProductTwoCoin (γ·R_b)/R_a, GeometricMeanTwoCoin
 *            ((γ·w_a)·R_b)/(w_b·R_a), UniV3 γ·q when a is its token 1, γ/q otherwise); NaNs are
 *            ignored; 0 when no pool of the pair is active.  Per call: rates depend on the state.
 *   screen   for each base p and each neighbour x of p: the pair score fl(r(p→x)·r(x→p)), and for
 *            every common neighbour y of p and x the triangle score, the larger of those of
 *            fl(fl(r(p→x)·r(x→y))·r(y→p)) and fl(fl(r(p→y)·r(y→x))·r(x→p)) that pass.  A score
 *            passes when > 1 − 2⁻⁴⁰.  The row's hubs are the first max_hubs passing triangles in
 *            (score descending, y ascending) order.  A row (p, x, hubs) is a candidate when its
 *            pair score or at least one triangle passes; candidates are ordered by (base index, x).
 *   solve    every candidate is quoted as cfmm_quote_arbitrage would quote it.
 *   select   the candidates that fill with profit >= min_profit[base], ordered by (base index,
 *            profit descending, x ascending); *found is their number.
 * The first min(*found, cap) rows are written: row_base, row_other, hub_count [cap], hubs
 * [cap × CFMM_ROUTE_MAX_HUBS] (1-based, best first, zero-padded), profit and price [cap].  The screen
 * is conservative: a profitable cycle's exact rate product exceeds 1, and the bests of a pool's two
 * directions multiply to γ² <= 1.  Passing rows to cfmm_execute_arbitrage with their minimum profits
 * closes the opportunities; each row is re-solved on the state the rows before it left, so rows that
 * share pools shrink or revert instead of spending twice.
 *
 * Before cfmm_finalize: CFMM_ERR_STATE.  q == 0 / nb == 0 do nothing (*found = 0).
 * CFMM_ERR_INVALID before anything runs for: rows: q < 0, a null base or other, tokens outside
 * 1..n_tokens or base == other, routed rows' hub rejections, a min_profit that is NaN, negative or
 * +inf.  Scan: nb < 0, cap < 0, a null found, base tokens outside 1..n_tokens or repeated, a
 * min_profit that is <= 0, NaN or Inf, max_hubs outside 0..CFMM_ROUTE_MAX_HUBS, a null base or
 * min_profit with nb > 0, a null output with cap > 0. */
int cfmm_quote_arbitrage(cfmm_ctx *ctx, int64_t q, const int64_t *base /* [q] */,
                         const int64_t *other /* [q] */, const int64_t *hub_off /* [q+1] */,
                         const int64_t *hubs /* [Σ] */, double *profit /* [q] */,
                         double *surplus_in /* [q] */, double *price /* [q] */,
                         uint8_t *status /* [q] */, double *hub_price /* [Σ] */,
                         double *hub_surplus /* [Σ] */, double *leg_delta /* [2L] */,
                         double *leg_lambda /* [2L] */);
int cfmm_execute_arbitrage(cfmm_ctx *ctx, int64_t q, const int64_t *base, const int64_t *other,
                           const double *min_profit /* [q] or NULL */, const int64_t *hub_off,
                           const int64_t *hubs, double *profit, double *surplus_in, double *price,
                           uint8_t *status, double *hub_price, double *hub_surplus,
                           double *leg_delta, double *leg_lambda);
int cfmm_scan_arbitrage(cfmm_ctx *ctx, int64_t nb, const int64_t *base /* [nb] */,
                        const double *min_profit /* [nb] */, int max_hubs, int64_t cap,
                        int64_t *found, int64_t *row_base /* [cap] */, int64_t *row_other /* [cap] */,
                        int64_t *hub_count /* [cap] */, int64_t *hubs /* [cap × 7] */,
                        double *profit /* [cap] */, double *price /* [cap] */);

/* ---- hub tokens chosen for order rows ----------------------------------------------------
 * For each order row (j = token_in[r], i = token_out[r], kind[r], amount[r], split orders' rules),
 * up to max_hubs (0..CFMM_ROUTE_MAX_HUBS) hub tokens for cfmm_quote_routed_orders /
 * cfmm_execute_routed_orders, ranked by the best single two-hop route through each.
 *   candidates  every token h that is a common neighbour of j and i in cfmm_scan_arbitrage's token
 *               adjacency (built on first use and kept with the pair index; it lists retired pools'
 *               pairs, so activity is read per call, from the pools), with allowed[h-1] != 0 when
 *               allowed [n_tokens] is given (NULL: every token).
 *   exact-in    (kind CFMM_SWAP_EXACT_IN, δ = amount) x_h = the largest f_k(δ) over the active pools
 *               k of {j, h} with j tendered, out_h = the largest f_k(x_h) over the active pools of
 *               {h, i} with h tendered.  f_k is the exact-input quote of one pool, cfmm_quote_swaps
 *               bit for bit (f_k(0) = 0); NaNs are ignored and a pair with no active pool gives 0.
 *               h is eligible when out_h > 0; rank out_h descending, then h ascending.
 *   exact-out   (kind CFMM_SWAP_EXACT_OUT, y = amount) c_h = the smallest x*_k(y) over the active
 *               pools of {h, i} with h tendered, in_h = the smallest x*_k(c_h) over the active pools
 *               of {j, h} with j tendered.  x*_k is cfmm_quote_swaps_exact_out's search, bit for bit;
 *               +inf (unreachable, or no active pool) propagates.  h is eligible when in_h is finite;
 *               rank in_h ascending, then h ascending.
 * Outputs: the first max_hubs eligible hubs in rank order, as packed CSR: hub_off [q+1] (hub_off[0]
 * = 0) and hubs [hub_off[q]] (1-based, at most q·max_hubs), ready for the routed calls, which use
 * them in the listed order; hub_score [hub_off[q]] (NULL: not written) = out_h or in_h; n_eligible
 * [q] (NULL: not written) = the eligible hubs before truncation.  A row with amount 0 gets no hubs
 * and n_eligible 0; max_hubs = 0 gives no hubs but still counts the eligible ones.  Max, min and the
 * ranking do not depend on the evaluation order, so the result is deterministic.
 *
 * The score is that of the best single route through h, not of h's share in an optimal split:
 * cfmm_quote_routed_orders then splits the row optimally over the direct pools and the chosen hubs'
 * pools.  Routes through two hubs or pools between hubs are not considered (cfmm_solve's).
 * Execute: pass the rows with these hubs to cfmm_execute_routed_orders.  The hubs are chosen once,
 * on the state at this call; the execute then re-solves each row on the state the earlier rows left.
 *
 * Synchronous; changes no state.  Before cfmm_finalize: CFMM_ERR_STATE.  CFMM_ERR_INVALID before
 * anything runs for every argument split orders reject, max_hubs outside 0..CFMM_ROUTE_MAX_HUBS, and
 * a null hub_off or hubs with q > 0.  q == 0 writes hub_off[0] = 0 (when given) and runs nothing. */
int cfmm_choose_order_hubs(cfmm_ctx *ctx, int64_t q, const int64_t *token_in /* [q] */,
                           const int64_t *token_out /* [q] */, const uint8_t *kind /* [q] */,
                           const double *amount /* [q] */, int max_hubs,
                           const uint8_t *allowed /* [n_tokens] or NULL */, int64_t *hub_off /* [q+1] */,
                           int64_t *hubs /* [q·max_hubs] */, double *hub_score /* [q·max_hubs] or NULL */,
                           int64_t *n_eligible /* [q] or NULL */);

/* ---- the best path of each order row through allowed tokens --------------------------------
 * For each order row (j = token_in[r], i = token_out[r], kind[r], amount[r], split orders' rules),
 * the best single path of at most H = max_hops (1..CFMM_PATH_MAX_HOPS) hops from j to i whose
 * intermediate tokens are in B, one pool per hop, as cfmm_execute_paths takes it.
 *   B           the tokens t with allowed[t-1] != 0 (allowed [n_tokens], required), minus j and i;
 *               at most CFMM_BEST_PATH_MAX_TOKENS per row.  A token of B can appear more than once
 *               in a path; j and i appear only at its ends.
 *   hops        a hop u → v uses one active pool of {u, v}: all three types, appended pools
 *               included, a pool stored with its tokens exchanged mapped back (the pools
 *               cfmm_pair_pools lists for {u, v}, retired ones skipped).  f_k is the exact-input
 *               quote of pool k (cfmm_quote_swaps bit for bit), x*_k the exact-out search
 *               (cfmm_quote_swaps_exact_out bit for bit), both on the state at this call.
 *   exact-in    (kind CFMM_SWAP_EXACT_IN, δ = amount) "at most h hops", level by level.  a₀(j) = δ;
 *               every other token is unreached.  For h = 1 … H−1 and u ∈ B, the candidates are
 *               f_k(a_{h−1}(u')) over every reached u' ∈ {j} ∪ B and every active pool k of {u', u}
 *               with u' tendered; a candidate counts only when it is > 0 (NaNs are ignored).
 *               a_h(u) is the best candidate when it is strictly greater than a_{h−1}(u), else
 *               a_{h−1}(u) (a reached u stays reached, j keeps δ).  The final hop's candidates are
 *               f_k(a_{H−1}(u)) over the active pools of {u, i}, u ∈ {j} ∪ B reached; the best is
 *               the path, its value the i received.
 *   exact-out   (kind CFMM_SWAP_EXACT_OUT, y = amount) the mirror image, backwards from i: c₀(i) = y;
 *               for u ∈ B the candidates are x*_k(c_{h−1}(v)) over reached v ∈ {i} ∪ B and the
 *               active pools k of {u, v} with u tendered, kept when finite; c_h(u) is the best when
 *               strictly smaller than c_{h−1}(u).  The final hop's candidates are x*_k(c_{H−1}(v))
 *               over the active pools of {j, v} with j tendered; the value is the j paid.
 *   ranking     candidates rank by the amount (larger exact-in, smaller exact-out), then fewer
 *               hops, then the smaller predecessor token (u' exact-in, v exact-out; j or i at the
 *               first hop of the DP), then the earlier position in {u', u}'s cfmm_pair_pools list.
 *               That is a total order, so the result does not depend on the evaluation order.
 * Outputs.  The walk is rebuilt from each level's predecessors, in path order j → … → i, as packed
 * CSR: hop_off [q+1] (hop_off[0] = 0; at most q·max_hops hops), hop_type / hop_pool (a pool as
 * cfmm_quote_paths addresses it) and hop_token (1-based, the token each hop delivers; the last is
 * i).  hop_tender / hop_received (NULL: not written) are the DP's amounts, which are cfmm_quote_paths'
 * hop_tender / hop_received on the returned path bit for bit (the same recursion: x_{h+1} = λ_h
 * exact-in, y_{h−1} = x_h exact-out).  value [q] (NULL: not written) = the i received (exact-in) or
 * the j paid (exact-out), 0 for a row without a path.  status [q] (NULL: not written):
 *   CFMM_ORDER_FILLED       a path was found (amount 0: no hops, value 0);
 *   CFMM_ORDER_UNREACHABLE  no path of at most max_hops hops through B: no hops;
 *   CFMM_PATH_REPEATS_POOL  the best walk holds a gaining cycle that uses one pool twice (under
 *                           quotes on the unchanged state, a cycle through B can gain); it is not
 *                           a path cfmm_execute_paths accepts, so no hops are written.
 * Execute: pass the rows with hops to cfmm_execute_paths (Python Router.execute_best_paths).  The
 * paths are found once, on the state at this call; the execute re-prices each path on the state
 * the earlier paths left.
 *
 * Synchronous; changes no state.  Before cfmm_finalize: CFMM_ERR_STATE.  CFMM_ERR_INVALID before
 * anything runs for every argument split orders reject, max_hops outside 1..CFMM_PATH_MAX_HOPS, a
 * null allowed, a row whose B holds more than CFMM_BEST_PATH_MAX_TOKENS tokens, and a null hop_off,
 * hop_type, hop_pool or hop_token with q > 0.  q == 0 writes hop_off[0] = 0 (when given) and runs
 * nothing. */
#define CFMM_BEST_PATH_MAX_TOKENS 1024
#define CFMM_PATH_REPEATS_POOL 4
int cfmm_find_order_paths(cfmm_ctx *ctx, int64_t q, const int64_t *token_in /* [q] */,
                          const int64_t *token_out /* [q] */, const uint8_t *kind /* [q] */,
                          const double *amount /* [q] */, int max_hops /* 1..CFMM_PATH_MAX_HOPS */,
                          const uint8_t *allowed /* [n_tokens], required */, int64_t *hop_off /* [q+1] */,
                          int *hop_type /* [q·max_hops] */, int64_t *hop_pool /* [q·max_hops] */,
                          int64_t *hop_token /* [q·max_hops] */, double *hop_tender /* [q·max_hops] or NULL */,
                          double *hop_received /* [q·max_hops] or NULL */, double *value /* [q] or NULL */,
                          uint8_t *status /* [q] or NULL */);

/* ---- every token's value against one root over the whole pool graph -------------------------
 * For each row r (a root S = root[r], 1-based; kind[r]; amount[r] finite and > 0), the best walk of at
 * most H = max_hops (1..CFMM_PATH_MAX_HOPS) hops between S and every token, one pool per hop: what
 * each token is worth in S at this size, as an executable path.  No cap on the tokens.
 *   allowed     a mask [n_tokens] (NULL: every token); only allowed tokens are reached.  The root is
 *               always allowed, is never a destination and so appears only at one end of a walk;
 *               every other token may repeat.
 *   hops        a hop u → v uses one active pool of {u, v}: the pools cfmm_find_order_paths uses (all
 *               three types, appended pools included, a pool stored with its tokens exchanged mapped
 *               back, retired pools skipped).  f_k and x*_k are cfmm_quote_swaps /
 *               cfmm_quote_swaps_exact_out bit for bit, on the state at this call.
 *   exact-in    (CFMM_SWAP_EXACT_IN, "spend δ = amount of S: how much of each token t") a₀(S) = δ,
 *               every other token unreached (0).  For h = 1 … H and allowed t != S the candidates are
 *               f_k(a_{h−1}(u)) over every reached u and every active pool k of {u, t} with u
 *               tendered; a candidate counts only when it is > 0 (NaNs are ignored).  a_h(t) is the
 *               best candidate when it is strictly greater than a_{h−1}(t), else a_{h−1}(t).
 *   exact-out   (CFMM_SWAP_EXACT_OUT, "receive y = amount of S: how much of each token t must be
 *               paid") the mirror image, backwards from S: c₀(S) = y, every other token unreached
 *               (+inf); the candidates for u are x*_k(c_{h−1}(v)) over reached v and the active pools
 *               k of {u, v} with u tendered, kept when finite; c_h(u) is the best when strictly
 *               smaller than c_{h−1}(u).
 *   ranking     by the amount (larger exact-in, smaller exact-out), then the smaller neighbour token
 *               (u exact-in, v exact-out), then the smaller global insertion index of the pool (within
 *               a pair, the order of its cfmm_pair_pools list): cfmm_find_order_paths' ranking without
 *               its "fewer hops" key.  Every candidate that can win at level h comes from a token that
 *               changed at level h−1, so it has exactly h hops: a candidate from an unchanged token
 *               repeats one of an earlier level, which the target's value already matches or beats,
 *               and cannot be strictly better.  The result therefore depends neither on the order the
 *               candidates are evaluated in nor on whether unchanged tokens are skipped; the device
 *               skips them (a level relaxes only the pools of the previous level's changed tokens)
 *               and stops once no token changed.
 *   against cfmm_find_order_paths  On a graph without gaining cycles through allowed tokens (every
 *               pool's marginal price agrees with one price vector, fees > 0) the value and walk of
 *               (S, t) are cfmm_find_order_paths(S, t, allowed, H)'s.  With a gaining cycle the two may
 *               differ: here t is also an intermediate of other walks and keeps the value the cycle
 *               gives it, where cfmm_find_order_paths never passes through its destination.
 * Outputs per (row, token), row-major [q·n_tokens]:
 *   value       a_H(t) exact-in (0 unreached), c_H(t) exact-out (+inf unreached); the root holds the
 *               row's amount.
 *   hops        (NULL: not written) the length of the best walk; 0 for the root and unreached tokens.
 *   status      (NULL: not written) CFMM_ORDER_FILLED: reached, and the walk uses distinct pools (the
 *               root: 0 hops); CFMM_ORDER_UNREACHABLE; CFMM_PATH_REPEATS_POOL: the best walk holds a
 *               gaining cycle through one pool twice, value still the DP's amount (as
 *               cfmm_find_order_paths' DP).
 * frontier [q·max_hops] (NULL: not written): the tokens whose value changed at level h = 1 … H.  A
 * row whose entry for h = H is 0 has converged: more hops would change nothing.
 * Paths on request: the n_req pairs (req_row[j] 0-based, req_token[j] 1-based) get their walks as
 * cfmm_execute_paths takes them, packed CSR: hop_off [n_req+1] (hop_off[0] = 0; at most
 * n_req·max_hops hops), hop_type / hop_pool (a pool as cfmm_quote_paths addresses it), hop_token (the
 * token each hop delivers, 1-based), hop_tender / hop_received (NULL: not written), and req_status
 * [n_req] (NULL: not written) as status above.  Exact-in walks run root → t (token_in = the root),
 * exact-out walks t → root (token_in = t).  The amounts are cfmm_quote_paths' on that CSR bit for bit
 * (the walk is priced by its code), and the path's end amount is value.  The root itself gives 0 hops
 * and FILLED; an unreached or REPEATS_POOL request gives no hops.
 * Rows run in groups sized to a workspace kept on the context (freed with it); a row's outputs do not
 * depend on the other rows of the call or their order.
 *
 * Synchronous; changes no state.  Single GPU.  Before cfmm_finalize: CFMM_ERR_STATE.  CFMM_ERR_INVALID
 * before anything runs for q < 0, n_req < 0, a root outside 1..n_tokens, a kind other than 0 or 1, an
 * amount that is NaN, infinite, 0 or negative, max_hops outside 1..CFMM_PATH_MAX_HOPS, a request row
 * outside 0..q−1 or token outside 1..n_tokens, a null root, kind, amount or value with q > 0, and a
 * null req_row, req_token, hop_off, hop_type, hop_pool or hop_token with n_req > 0.  q == 0 writes
 * hop_off[0] = 0 (when given) and runs nothing. */
int cfmm_quote_token_values(cfmm_ctx *ctx, int64_t q, const int64_t *root /* [q] */,
                            const uint8_t *kind /* [q] */, const double *amount /* [q] */,
                            int max_hops /* 1..CFMM_PATH_MAX_HOPS */,
                            const uint8_t *allowed /* [n_tokens] or NULL */,
                            double *value /* [q·n_tokens] */, uint8_t *hops /* [q·n_tokens] or NULL */,
                            uint8_t *status /* [q·n_tokens] or NULL */,
                            int64_t *frontier /* [q·max_hops] or NULL */, int64_t n_req,
                            const int64_t *req_row /* [n_req] */, const int64_t *req_token /* [n_req] */,
                            int64_t *hop_off /* [n_req+1] */, int *hop_type /* [n_req·max_hops] */,
                            int64_t *hop_pool /* [n_req·max_hops] */,
                            int64_t *hop_token /* [n_req·max_hops] */,
                            double *hop_tender /* [n_req·max_hops] or NULL */,
                            double *hop_received /* [n_req·max_hops] or NULL */,
                            uint8_t *req_status /* [n_req] or NULL */);

/* ---- best paths and token values net of a per-hop cost ---------------------------------------
 * cfmm_find_order_paths and cfmm_quote_token_values rank walks by amount alone, so a hop that adds
 * one ulp wins.  On a chain each hop costs gas.  The _net calls return, per row (best paths) or per
 * (row, token) (token values), the result whose amount net of a fixed cost per hop is best.
 *   definition  P_L is the existing call's result with max_hops = L.  For L = 1 … H:
 *               eligible  P_L is CFMM_ORDER_FILLED;
 *               net       exact-in net_L = v_L − n_L·κ, exact-out net_L = v_L + n_L·κ (v_L the value,
 *                         n_L the hops, κ the hop cost), one IEEE multiply and then one IEEE add or
 *                         subtract, no fma;
 *               selection the eligible L with the best net: larger exact-in, smaller exact-out; on a
 *                         tie the larger L.
 *               Outputs are P_L's: hops, amounts, walk and value, and net.  No eligible L: P_H as it
 *               is, with net = value.  The root, and a row of amount 0, keep their outputs, with
 *               net = value.  κ = +inf is allowed (no walk into that token pays for itself): every
 *               n >= 1 nets ∓inf, so the tie rule gives the largest filled L, P_H when it fills.
 *   exactness   Each level's predecessors are kept, and a winner at level h has exactly h hops.  If the
 *               best walk W* by net has k hops and amount A*, P_k amounts to at least A* with at most k
 *               hops, so its net is at least A* − k·κ (exact-in; the mirror image exact-out).  The
 *               selection over L is therefore the optimum over every walk the DP ranks.
 *   κ = 0       Outputs are the existing call's bit for bit wherever the selection picks L = H.  It
 *               picks a shorter L only when (a) the existing call reports CFMM_PATH_REPEATS_POOL at H
 *               and a shorter L fills, or (b) rounding makes a shorter walk's quote strictly better:
 *               fl(f) need not be monotone in its input even though f is.  Both are improvements.
 *   limits      The costs are charged at the end, in the destination's units: intermediates are not
 *               charged, and costs that depend on the pool type (UniV3 tick crossings) are not modelled.
 *               The DP stays the existing one; the hop count is only a tie-break of its ranking, so a
 *               walk that is worse by amount but shorter is found only when it is some level's best.
 * cfmm_find_order_paths_net  cfmm_find_order_paths' arguments, plus hop_cost [q]: row r's κ in its
 *               settlement token (the token_out exact-in, the token_in exact-out), and net [q] (NULL: not
 *               written).  The final pass runs after every level of the DP instead of once: up to H
 *               final passes per row.
 * cfmm_quote_token_values_net  cfmm_quote_token_values' arguments, plus hop_cost [n_tokens]: κ_t, the
 *               cost of one hop in units of token t, shared by every row, and net [q·n_tokens] (NULL:
 *               not written).  The requested walks are those of the selected level.  frontier is the
 *               DP's, unchanged.  One more per-(row, token) pass per level; the workspace holds 17 more
 *               bytes per (row, token), so groups can be smaller.
 * Costs in every token: cfmm_quote_token_values (exact-in) rooted at the gas token with the gas of one
 * hop as its amount gives what a hop costs in each token (Python Router.hop_costs).
 *
 * Synchronous; change no state.  CFMM_ERR_INVALID before anything runs for every argument the existing
 * call rejects, and for a null hop_cost (token values: always; best paths: with q > 0) or a hop_cost
 * that is NaN or negative. */
int cfmm_find_order_paths_net(cfmm_ctx *ctx, int64_t q, const int64_t *token_in /* [q] */,
                              const int64_t *token_out /* [q] */, const uint8_t *kind /* [q] */,
                              const double *amount /* [q] */, int max_hops /* 1..CFMM_PATH_MAX_HOPS */,
                              const uint8_t *allowed /* [n_tokens], required */,
                              const double *hop_cost /* [q] */, int64_t *hop_off /* [q+1] */,
                              int *hop_type /* [q·max_hops] */, int64_t *hop_pool /* [q·max_hops] */,
                              int64_t *hop_token /* [q·max_hops] */,
                              double *hop_tender /* [q·max_hops] or NULL */,
                              double *hop_received /* [q·max_hops] or NULL */, double *value /* [q] or NULL */,
                              uint8_t *status /* [q] or NULL */, double *net /* [q] or NULL */);
int cfmm_quote_token_values_net(cfmm_ctx *ctx, int64_t q, const int64_t *root /* [q] */,
                                const uint8_t *kind /* [q] */, const double *amount /* [q] */,
                                int max_hops /* 1..CFMM_PATH_MAX_HOPS */,
                                const uint8_t *allowed /* [n_tokens] or NULL */,
                                const double *hop_cost /* [n_tokens] */, double *value /* [q·n_tokens] */,
                                uint8_t *hops /* [q·n_tokens] or NULL */,
                                uint8_t *status /* [q·n_tokens] or NULL */, double *net /* [q·n_tokens] or NULL */,
                                int64_t *frontier /* [q·max_hops] or NULL */, int64_t n_req,
                                const int64_t *req_row /* [n_req] */, const int64_t *req_token /* [n_req] */,
                                int64_t *hop_off /* [n_req+1] */, int *hop_type /* [n_req·max_hops] */,
                                int64_t *hop_pool /* [n_req·max_hops] */,
                                int64_t *hop_token /* [n_req·max_hops] */,
                                double *hop_tender /* [n_req·max_hops] or NULL */,
                                double *hop_received /* [n_req·max_hops] or NULL */,
                                uint8_t *req_status /* [n_req] or NULL */);

/* ---- orders routed over every pool among their allowed tokens ------------------------------
 * A row sells δ = amount[r] of j = token_in[r] for i = token_out[r] (1-based, distinct; exact-in:
 * exact-out rows are below) over every pool among j, i and the allowed tokens, split optimally: route! with
 * Swap(i, j, δ) (src/objectives.jl:106-146) restricted to the row's pools, one convex dual per row.
 *   B        the tokens t with allowed[t-1] != 0 (allowed [n_tokens], required), minus j and i; at
 *            most CFMM_SUBGRAPH_MAX_TOKENS per row.  One mask per call (a list per row: the _rows
 *            calls, "per-row masks" below).
 *   T        the tokens of {j, i} ∪ B connected to i through active pools whose two tokens both lie
 *            in {j, i} ∪ B.  Pools in a component cut off from i would only trade at ν ≈ √eps.
 *   pools    every pool of every pair inside T: all three types, appended pools included, retired
 *            pools listed (they trade (0, 0)), in global insertion order (cfmm_num_pools' numbering).
 *   tokens   local order: i, j, then B ∩ T ascending.  A row with j ∉ T (amount > 0) is
 *            CFMM_ORDER_UNREACHABLE; it still lists T (without j) and its pools, with zero legs.
 * Problem.  Minimise g(ν) = δ·ν_j + Σ_k π_k(ν) over the row's pools k on the box ν_i >= 1 + √eps,
 * ν_t >= √eps otherwise (no upper bound), π_k(ν) = ν_a·(Λ_a − Δ_a) + ν_b·(Λ_b − Δ_b) at the pool's
 * legs.  A pool's legs at ν are split orders' (find_arb! of the materialising sweep at ν taken at
 * the pool's stored tokens, split_legs; cfmm_sweep with materialize = 1 gives the same bits).
 * Sums, in fixed orders with no atomics, so a row's result does not depend on the batch:
 *   Ψ_t      over the row's pools that hold t, in pool order, split orders' warp tree (partial l adds
 *            the entries ≡ l (mod 32) from +0.0, then the xor butterfly 16 … 1); each entry is one
 *            IEEE subtraction Λ_t − Δ_t.  The gradient is (δ at j, 0 elsewhere) + Ψ.
 *   value    thread l of 256 adds the terms of pools ≡ l (mod 256) from +0.0 (each term
 *            ν_a·c_a + ν_b·c_b, IEEE), the xor butterfly in each warp, then the 8 warps in order;
 *            g = δ·ν_j + that sum.
 * Optimizer: cfmm_solve's projected L-BFGS (m = 5; its two-loop recursion over [S Y pg], Armijo
 * backtracking with its noise slack, its restart rule and its factr test on two consecutive steps;
 * the control code is shared), run by one CTA per row with every vector in shared memory.
 *   start    ν_i = 1; then breadth-first rounds over the active pools: a token not yet priced gets
 *            the largest r(a → b)·ν_b over its pools to tokens priced in earlier rounds (r:
 *            cfmm_scan_arbitrage's rate of one pool), and keeps it; then clamped to the box.
 *   stop     pg = cfmm_solve's clipped projected gradient, m_r = max_t ν_t·|pg_t| / (δ·ν_j), each
 *            token's imbalance valued at its price relative to the order's value.  Status 0 when
 *            m_r <= rtol; 1 (relative decrease <= factr·eps twice, or no move), 2 (max_iter),
 *            3 (max_fun), 4 (line search failed) and 5 (NaN) as cfmm_solve.
 * What a fill promises.  A row is CFMM_ORDER_FILLED only at solver status 0; otherwise it is
 * CFMM_ORDER_NOT_CONVERGED, keeps its m_r and solver status, and its legs, paid and received read
 * 0.  A filled row has received = Ψ_i, paid = −Ψ_j (within rtol·δ of δ when ν_j is off its bound),
 * every intermediate's net Ψ_b >= −rtol·δ·ν_j/ν_b, and a duality gap of at most |T|·rtol·δ·ν_j plus
 * the box's √eps terms.  Amount 0 fills with zeros and runs no solve.  Non-finite legs (a
 * GeometricMean closed form that overflows): a line-search trial that meets one backs off and the
 * row goes on, so it may still fill from finite iterates; a row whose committed iterate holds one
 * (its reported Ψ or m_r not finite) ends CFMM_ORDER_NOT_CONVERGED, as in every row kind below.
 * Outputs (cfmm_subgraph_out; every pointer may be NULL):
 *   per row  paid, received, status (CFMM_ORDER_*), solver_status (−1 when no solve ran),
 *            iterations, fun_evals, merit (m_r; 0 without a solve);
 *   tokens   tok_off [q+1]; token (1-based), nu, psi [tok_off[q]] in local order, written when
 *            tok_off[q] <= tok_cap (ν and Ψ at the last iterate, 0 without a solve);
 *   legs     leg_off [q+1]; leg_type, leg_pool (a pool as cfmm_quote_swaps takes it), leg_delta,
 *            leg_lambda ([2L], (Δ, Λ) in ingest token order as cfmm_get_trades lays them out) in
 *            the row's pool order, written when leg_off[q] <= leg_cap; 0 unless filled.
 *   Ask a quote with tok_cap = leg_cap = 0 for the sizes first, as with cfmm_pair_pools.
 * cfmm_quote_subgraph_orders prices every row on the current state on its own; no state changes.
 * cfmm_execute_subgraph_orders runs the rows in batch order, each re-solved on the state the earlier
 * filled rows left.  limit (NULL: none) is the minimum received; an equal limit fills, a smaller
 * received reverts with CFMM_ORDER_LIMIT.  A filled row applies split_leg's transition at its ν to
 * each active pool (two-coin R <- (R + γΔ) − Λ; UniV3 the q′ rule, current tick updated), then the
 * bookkeeping of cfmm_execute_swaps runs (state version, guard-free flag, fixed-point scale, UniV3
 * tick records); the materialised trades stay.  Two rows conflict when they share a token of
 * {j, i} ∪ B; rows are leveled by cfmm_execute_paths' rule, one launch per level.  With one mask per
 * call, rows with a non-empty B share its tokens and run one after another (per-row masks, below, let
 * rows on disjoint tokens share a level).  An execute whose token
 * or leg outputs are given with a cap below the size is rejected before anything changes.
 * Options (cfmm_subgraph_opts, NULL: max_iter 1000, max_fun 4000, rtol 1e-4, factr 0: the factr test
 * then stops only after two steps that do not lower g).  The observed floor of m_r on random
 * markets whose pools disagree on prices is 1e-9 .. 1e-5 per row (see DESIGN §4.5).
 * Synchronous.  Before cfmm_finalize: CFMM_ERR_STATE.  q == 0 does nothing.  CFMM_ERR_INVALID before
 * anything runs for: q < 0, a null token_in, token_out or amount; tokens outside 1..n_tokens or
 * token_in == token_out; an amount that is NaN, Inf or negative; a null allowed; a row whose B holds
 * more than CFMM_SUBGRAPH_MAX_TOKENS tokens; max_iter or max_fun < 1, rtol not finite and > 0,
 * factr not finite and >= 0; a limit that is NaN, negative or +inf. */
#define CFMM_SUBGRAPH_MAX_TOKENS 256
#define CFMM_ORDER_NOT_CONVERGED 5
typedef struct {
  int max_iter, max_fun;
  double rtol, factr;
} cfmm_subgraph_opts;
typedef struct {
  double *paid, *received;                       /* [q] */
  uint8_t *status;                               /* [q] */
  int *solver_status, *iterations, *fun_evals;   /* [q] */
  double *merit;                                 /* [q] */
  int64_t *tok_off;                              /* [q+1] */
  int64_t tok_cap;
  int64_t *token;                                /* [tok_off[q]] */
  double *nu, *psi;                              /* [tok_off[q]] */
  int64_t *leg_off;                              /* [q+1] */
  int64_t leg_cap;
  int *leg_type;                                 /* [leg_off[q]] */
  int64_t *leg_pool;                             /* [leg_off[q]] */
  double *leg_delta, *leg_lambda;                /* [2·leg_off[q]] */
} cfmm_subgraph_out;
int cfmm_quote_subgraph_orders(cfmm_ctx *ctx, int64_t q, const int64_t *token_in /* [q] */,
                               const int64_t *token_out /* [q] */, const double *amount /* [q] */,
                               const uint8_t *allowed /* [n_tokens], required */,
                               const cfmm_subgraph_opts *opts /* NULL = defaults */,
                               cfmm_subgraph_out *out);
int cfmm_execute_subgraph_orders(cfmm_ctx *ctx, int64_t q, const int64_t *token_in,
                                 const int64_t *token_out, const double *amount,
                                 const double *limit /* [q] or NULL */, const uint8_t *allowed,
                                 const cfmm_subgraph_opts *opts, cfmm_subgraph_out *out);

/* ---- subgraph orders of either kind: exact-in and exact-out rows ----------------------------
 * cfmm_quote_subgraph_swap_orders / cfmm_execute_subgraph_swap_orders take the arguments of the two
 * calls above plus kind [q] (NULL: every row exact-in).  A row of kind CFMM_SWAP_EXACT_IN is the
 * subgraph order above, bit for bit; cfmm_quote_subgraph_orders and cfmm_execute_subgraph_orders
 * are these calls with kind = NULL.  A row of kind CFMM_SWAP_EXACT_OUT buys y = amount[r] of
 * i = token_out[r] and pays in j = token_in[r], over the same B, T, pools and local token order
 * (i, j, then B ∩ T), legs, sums, optimizer and CTA reduction as an exact-in row.
 * Problem.  The primal is: maximise Ψ_j subject to Ψ_i >= y and Ψ_t >= 0 for every other t in T.
 * Its dual: minimise g(ν) = −y′·ν_i + Σ_k π_k(ν) on the box ν_j = 1 (lower = upper = 1), ν_t >= √eps
 * for every other t (i included), with y′ = y·(1 + rtol) rounded up (fma, round toward +inf).  ν_j is
 * fixed because the optimal value, −paid, is negative and g is positively homogeneous: with only a
 * lower bound, scaling ν up would drive g to −∞.  The gradient is (−y′ at i, 0 elsewhere) + Ψ; the
 * value is −y′·ν_i + the pool sum of exact-in rows.
 *   start    ν_j = 1; then the breadth-first pricing of exact-in rows from j instead of i; then
 *            clamped to the box.
 *   box      slot j is clamped to [1, 1], so pg_j = 0 and its step is 0; every other slot uses the
 *            lower-bound clip of exact-in rows.
 *   stop     m_r = max_t ν_t·|pg_t| / (y·ν_i), the imbalance valued against the order's value in j.
 *            Status 0 when m_r <= rtol; the other statuses as for exact-in rows.  Since
 *            |pg_i| = |Ψ_i − y′| <= rtol·y at the stop, a converged row receives at least y.
 * Capacity, checked once per row after its pool list is built and before any solve.  C_i is the sum,
 * over the row's active pools holding i in pool order (per thread, then sg's CTA sum), of what the
 * pool could ever pay out of i: a two-coin pool's reserve R_i; a UniV3 pool's walk to the end of its
 * ladder (f(DBL_MAX) of cfmm_quote_swaps_exact_out, the quantity of its unreachable case).  A row is
 * CFMM_ORDER_UNREACHABLE when j ∉ T or y >= C_i.  A row that passes this check but still cannot be
 * served (for example i reachable only behind a thin intermediate pool) has an unbounded dual: it
 * ends at max_iter, max_fun or NaN and is CFMM_ORDER_NOT_CONVERGED, trading nothing.
 * What a fill promises.  A row fills only at solver status 0 and received >= y; a status-0 row whose
 * received is below y (rounding) is CFMM_ORDER_NOT_CONVERGED with solver_status 0.  A filled row has
 * received = Ψ_i in [y, y·(1 + 2·rtol)] when ν_i is off its bound, paid = −Ψ_j, every intermediate
 * Ψ_b >= −rtol·y·ν_i/ν_b, and a duality gap of at most |T|·rtol·y·ν_i plus the box's √eps terms.
 * Amount 0 fills with zeros and runs no solve.  The outputs are those of cfmm_subgraph_out.
 * Execute.  limit (NULL: none) is the maximum paid for an exact-out row (+inf allowed; an equal limit
 * fills, paid > limit reverts with CFMM_ORDER_LIMIT) and the minimum received for an exact-in row.
 * The transition, bookkeeping, conflict rule and levels are those of exact-in rows; a level runs its
 * exact-in rows and its exact-out rows as two launches (they share no token).  A quote runs the
 * exact-in rows and the exact-out rows as two launches.
 * Errors: those of the calls above, and CFMM_ERR_INVALID before anything runs for a kind other than
 * CFMM_SWAP_EXACT_IN or CFMM_SWAP_EXACT_OUT, an exact-in limit that is NaN, negative or +inf, and an
 * exact-out limit that is NaN or negative. */
int cfmm_quote_subgraph_swap_orders(cfmm_ctx *ctx, int64_t q, const int64_t *token_in /* [q] */,
                                    const int64_t *token_out /* [q] */,
                                    const uint8_t *kind /* [q] or NULL: all exact-in */,
                                    const double *amount /* [q] */,
                                    const uint8_t *allowed /* [n_tokens], required */,
                                    const cfmm_subgraph_opts *opts /* NULL = defaults */,
                                    cfmm_subgraph_out *out);
int cfmm_execute_subgraph_swap_orders(cfmm_ctx *ctx, int64_t q, const int64_t *token_in,
                                      const int64_t *token_out,
                                      const uint8_t *kind /* [q] or NULL: all exact-in */,
                                      const double *amount, const double *limit /* [q] or NULL */,
                                      const uint8_t *allowed, const cfmm_subgraph_opts *opts,
                                      cfmm_subgraph_out *out);

/* ---- token baskets liquidated over every pool among their allowed tokens --------------------
 * A row sells a basket of tokens for i = token_out[r] over every pool among i, the basket and the
 * allowed tokens, split optimally: route! with BasketLiquidation(i, Δin) (src/objectives.jl)
 * restricted to the row's pools, one convex dual per row.  A subgraph order (above) is the basket
 * of one entry: a one-entry basket row gives that call's outputs bit for bit.
 *   basket   entries basket_off[r] .. basket_off[r+1] − 1 of basket_token (1-based) and
 *            basket_amount (δ_k, finite and >= 0): 1 to CFMM_BASKET_MAX_TOKENS entries, distinct, none
 *            of them i.  basket_off [q+1] starts at 0 and does not decrease.
 *   B        the allowed tokens (allowed [n_tokens], required; one mask per call) minus i and the
 *            basket.  A row's tokens other than i (basket ∪ B) number at most
 *            CFMM_SUBGRAPH_MAX_TOKENS + 1.
 *   T        the tokens of {i} ∪ basket ∪ B connected to i through active pools whose two tokens both
 *            lie in that set.  An entry with δ_k > 0 outside T makes the row CFMM_ORDER_UNREACHABLE;
 *            an entry with δ_k = 0 outside T is dropped from the row's tokens.
 *   pools    every pool of every pair inside T, in global insertion order, as for subgraph orders.
 *   tokens   local order: i, then the basket entries in T in the caller's order, then B ∩ T ascending.
 * Problem.  Minimise g(ν) = Σ_k δ_k·ν_k + Σ_p π_p(ν) on the box of Swap (ν_i >= 1 + √eps, ν_t >= √eps
 * otherwise).  Legs, sums, optimizer and start are those of subgraph orders, with the gradient
 * (δ_k at b_k, 0 elsewhere) + Ψ and V = Σ_k δ_k·ν_k added in basket order (the first term alone).
 *   stop     m_r = max_t ν_t·|pg_t| / V; status 0 when m_r <= rtol.
 * What a fill promises.  A row fills only at solver status 0 (else CFMM_ORDER_NOT_CONVERGED, with
 * zero legs, paid and received).  A filled row has received = Ψ_i and paid_k = −Ψ_{b_k}: each basket
 * token is paid within rtol·V/ν_k of δ_k when ν_k is off its bound; every intermediate's net is
 * Ψ_b >= −rtol·V/ν_b; and the duality gap is at most |T|·rtol·V plus the box's √eps terms.  A row
 * whose amounts are all 0 fills with zeros and runs no solve.
 * Outputs (cfmm_basket_out; every pointer may be NULL): those of cfmm_subgraph_out, except that paid
 * has one entry per basket entry ([basket_off[q]], 0 for an entry outside T); received and the rest
 * are per row.  Ask a quote with tok_cap = leg_cap = 0 for the sizes first.
 * cfmm_quote_basket_orders prices every row on the current state on its own; no state changes.
 * cfmm_execute_basket_orders runs the rows in batch order, each re-solved on the state the earlier
 * filled rows left; limit (NULL: none) is the minimum received of i, and an equal limit fills.  A
 * filled row applies split_leg's transition, then the bookkeeping of cfmm_execute_swaps.  Two rows
 * conflict when they share a token of {i} ∪ basket ∪ B; rows are leveled by cfmm_execute_paths'
 * rule, one launch per level (with an empty mask, rows on disjoint tokens run in one launch).  An
 * execute whose token or leg outputs are given with a cap below the size is rejected before
 * anything changes.
 * Options: cfmm_subgraph_opts, with the same defaults.  Synchronous.  Before cfmm_finalize:
 * CFMM_ERR_STATE.  q == 0 does nothing.  CFMM_ERR_INVALID before anything runs for: the argument
 * errors of subgraph orders (q, a null array, the mask, the options, amounts, limits); token_out or
 * a basket token outside 1..n_tokens; basket_off[0] != 0 or a decreasing basket_off; an empty basket
 * or one longer than CFMM_BASKET_MAX_TOKENS; a basket token that appears twice or equals token_out;
 * a row with more than CFMM_SUBGRAPH_MAX_TOKENS + 1 tokens besides token_out. */
#define CFMM_BASKET_MAX_TOKENS 16
typedef struct {
  double *paid;                                  /* [basket_off[q]] */
  double *received;                              /* [q] */
  uint8_t *status;                               /* [q] */
  int *solver_status, *iterations, *fun_evals;   /* [q] */
  double *merit;                                 /* [q] */
  int64_t *tok_off;                              /* [q+1] */
  int64_t tok_cap;
  int64_t *token;                                /* [tok_off[q]] */
  double *nu, *psi;                              /* [tok_off[q]] */
  int64_t *leg_off;                              /* [q+1] */
  int64_t leg_cap;
  int *leg_type;                                 /* [leg_off[q]] */
  int64_t *leg_pool;                             /* [leg_off[q]] */
  double *leg_delta, *leg_lambda;                /* [2·leg_off[q]] */
} cfmm_basket_out;
int cfmm_quote_basket_orders(cfmm_ctx *ctx, int64_t q, const int64_t *token_out /* [q] */,
                             const int64_t *basket_off /* [q+1] */,
                             const int64_t *basket_token /* [basket_off[q]] */,
                             const double *basket_amount /* [basket_off[q]] */,
                             const uint8_t *allowed /* [n_tokens], required */,
                             const cfmm_subgraph_opts *opts /* NULL = defaults */, cfmm_basket_out *out);
int cfmm_execute_basket_orders(cfmm_ctx *ctx, int64_t q, const int64_t *token_out,
                               const int64_t *basket_off, const int64_t *basket_token,
                               const double *basket_amount, const double *limit /* [q] or NULL */,
                               const uint8_t *allowed, const cfmm_subgraph_opts *opts,
                               cfmm_basket_out *out);

/* ---- token baskets bought and sold together: basket rows with bought entries -----------------
 * cfmm_quote_basket_swap_orders / cfmm_execute_basket_swap_orders take the arguments of the two
 * calls above plus entry_kind [basket_off[q]] (NULL: every entry sold).  An entry of kind
 * CFMM_SWAP_EXACT_IN sells up to δ_k = basket_amount[k] of b_k; one of kind CFMM_SWAP_EXACT_OUT buys
 * y_l = basket_amount[l] of b_l.  Every row settles in i = token_out[r].  A row whose entries are all
 * sold is a basket row above, bit for bit and with the same launches.  A row with at least one bought
 * entry is a buy row: it has the same B, T, reachability rule (an entry with a positive amount outside
 * T makes the row CFMM_ORDER_UNREACHABLE; a zero entry outside T is dropped), pools, legs, sums,
 * optimizer and CTA reduction, with:
 *   tokens   local order: the bought entries in T in the caller's order, then i, then the sold
 *            entries in T in the caller's order, then B ∩ T ascending.  With one bought entry and no
 *            sold entry this is the exact-out subgraph row's order (i, j, B ∩ T).
 * Problem.  The primal is: maximise Ψ_i (it may be negative: the row pays on net) subject to
 * Ψ_k >= −δ_k for sold entries, Ψ_l >= y_l for bought entries and Ψ_t >= 0 for every other t in T.
 * Its dual: minimise g(ν) = Σ_k δ_k·ν_k − Σ_l y′_l·ν_l + Σ_p π_p(ν) on the box ν_i = 1 (lower = upper
 * = 1), ν_t >= √eps for every other t, with y′ = y·(1 + rtol) rounded up as exact-out rows do.  ν_i is
 * fixed for the reason it is fixed in exact-out rows.  The gradient is lin + Ψ, lin = δ at sold
 * entries, −y′ at bought entries and 0 elsewhere; the value is Σ lin_e·ν_e over the entries in local
 * order (the first term alone) plus the pool sum.
 *   start    ν_i = 1; the breadth-first pricing of subgraph rows from i's slot; clamped to the box.
 *   stop     V = Σ_e amount_e·ν_e over the entries in local order (y, not y′);
 *            m_r = max(max_t ν_t·|pg_t| / V, max over bought l with y_l > 0 of ν_l·|pg_l| / (y_l·ν_l)).
 *            The second term holds each bought entry to rtol·y_l even when the sold entries dominate
 *            V.  Status 0 when m_r <= rtol.
 * Capacity, checked once per row before any solve: for each bought entry with y_l > 0, C_l is the
 * exact-out rule's capacity at b_l over the row's pools.  The row is CFMM_ORDER_UNREACHABLE when
 * y_l >= C_l for some l.  A row that passes this check but cannot be served has an unbounded dual and
 * ends CFMM_ORDER_NOT_CONVERGED, trading nothing.
 * What a fill promises.  A buy row fills only at solver status 0 with Ψ_l >= y_l for every bought
 * entry with y_l > 0 (a status-0 row short of one is CFMM_ORDER_NOT_CONVERGED with solver_status 0).
 * A filled row has: received = Ψ_i (negative when the row pays on net); paid_k = −Ψ_{b_k}, so a
 * bought entry reads paid_l = −Ψ_l <= −y_l; each sold entry paid within rtol·V/ν_k of δ_k when ν_k is
 * off its bound; each bought entry receiving Ψ_l in [y_l, y_l·(1 + 2·rtol)] when ν_l is off its bound;
 * every other token (an intermediate, or a bought entry with y_l = 0) Ψ_b >= −rtol·V/ν_b; and a
 * duality gap of at most |T|·rtol·V plus the box's √eps terms.  A row whose amounts are all 0 fills
 * with zeros and runs no solve.  The outputs are those of cfmm_basket_out.
 * Execute.  limit (NULL: none) is the minimum Ψ_i.  For a buy row it may be negative (pay at most
 * −limit) or −inf; an equal limit fills and a smaller Ψ_i reverts with CFMM_ORDER_LIMIT.  A sell-only
 * row's limit follows cfmm_execute_basket_orders.  The transition, bookkeeping, conflict rule
 * ({i} ∪ entries ∪ B) and levels are those of basket rows; a level runs its sell-only rows and its
 * buy rows as two launches (they share no token).  A quote runs the sell-only rows and the buy rows
 * as two launches.
 * Errors: those of the basket calls, and CFMM_ERR_INVALID before anything runs for an entry kind
 * other than CFMM_SWAP_EXACT_IN or CFMM_SWAP_EXACT_OUT, and a buy row's limit that is NaN or +inf. */
int cfmm_quote_basket_swap_orders(cfmm_ctx *ctx, int64_t q, const int64_t *token_out /* [q] */,
                                  const int64_t *basket_off /* [q+1] */,
                                  const int64_t *basket_token /* [basket_off[q]] */,
                                  const uint8_t *entry_kind /* [basket_off[q]] or NULL: every entry sold */,
                                  const double *basket_amount /* [basket_off[q]] */,
                                  const uint8_t *allowed /* [n_tokens], required */,
                                  const cfmm_subgraph_opts *opts /* NULL = defaults */,
                                  cfmm_basket_out *out);
int cfmm_execute_basket_swap_orders(cfmm_ctx *ctx, int64_t q, const int64_t *token_out,
                                    const int64_t *basket_off, const int64_t *basket_token,
                                    const uint8_t *entry_kind /* [basket_off[q]] or NULL */,
                                    const double *basket_amount, const double *limit /* [q] or NULL */,
                                    const uint8_t *allowed, const cfmm_subgraph_opts *opts,
                                    cfmm_basket_out *out);

/* ---- limit orders: sell up to an amount at no worse than a limit price, filled partially -----
 * cfmm_quote_limit_orders / cfmm_execute_limit_orders take the basket calls' arguments plus
 * limit_price [basket_off[q]].  Row r settles in i = token_out[r]; entry k sells up to
 * δ_k = basket_amount[k] of b_k (finite, >= 0) for as long as the margin pays at least
 * c_k = limit_price[k] of i per unit of b_k (finite, >= 0).  B, T, pools, legs, sums, optimizer,
 * options and CTA reduction are those of basket rows (one allowed mask per call), with:
 *   reach    an entry outside T with c_k > 0 cannot fill at any price: it is dropped and paid 0.  An
 *            entry outside T with c_k = 0 follows the basket rule: δ_k > 0 makes the row
 *            CFMM_ORDER_UNREACHABLE.  A row whose remaining amounts are all 0 fills with zeros and
 *            runs no solve.
 *   tokens   local order: i, then the entries in T in the caller's order, then B ∩ T ascending.
 * Buying with a budget is the same row with the roles swapped: settle in the bought token, sell the
 * budget token, and set c = 1 / (the highest price paid per unit bought).  Buys capped at a bought
 * quantity are not offered (their conjugate is piecewise linear in ν).
 * Problem.  The primal is: maximise S = Ψ_i + Σ_k c_k·Ψ_k subject to Ψ_k >= −δ_k at the entries and
 * Ψ_t >= 0 for every other t in T (i included).  Its conjugate is finite only on ν_i >= 1, ν_k >= c_k,
 * ν_t >= 0, where it is Σ_k δ_k·(ν_k − c_k), so the dual is
 *   g(ν) = Σ_k δ_k·ν_k − Σ_k δ_k·c_k + Σ_p π_p(ν),
 * the basket row's dual with each entry's lower bound raised to its limit, plus a constant.  The device
 * minimises it without the constant on the box
 *   ν_i >= 1 + √eps (Swap's), ν_k >= lo_k = fmax(c_k, √eps) (one IEEE operation: a zero limit gives the
 *   basket bound bit for bit), ν_t >= √eps for every other token,
 * with lin = δ_k at the entries.  The value, V = Σ_k δ_k·ν_k and m_r = max_t ν_t·|pg_t| / V are the
 * basket row's, in the same operation order; status 0 when m_r <= rtol.
 *   start    the basket row's breadth-first pricing from i, clamped to this box.
 * Complementary slackness gives the limit-order reading: an entry whose ν_k is above its bound sells
 * in full (Ψ_k = −δ_k up to the stop); an entry that sells partially has ν_k on c_k, so its last unit
 * sold at the limit rate (within the box's √eps).  With every c_k = 0 a row is a basket row: the same
 * outputs bit for bit.
 * What a fill promises.  A row fills only at solver status 0 (else CFMM_ORDER_NOT_CONVERGED, trading
 * nothing).  A filled row has received = Ψ_i and paid_k = −Ψ_{b_k} with:
 *   each paid_k <= δ_k + rtol·V/ν_k (Ψ_k + δ_k is the gradient, within rtol·V/ν_k of 0 off the
 *   bound and at least −rtol·V/ν_k on it); an entry with ν_k off its bound sells in full, within
 *   rtol·V/ν_k of δ_k.  paid_k < 0 (the row receives b_k) happens only with ν_k on its bound: the
 *   primal values b_k at c_k, so when the pools deliver b_k for less than that (through the row's other
 *   entries, or a cycle), receiving it raises S.  A single entry over pools with no cycle never does;
 *   every intermediate's net Ψ_b >= −rtol·V/ν_b;
 *   the surplus S = received − Σ_k c_k·paid_k >= −(|T|·rtol·V + Σ_{t on its bound}
 *   (lo_t − c_t)·max(Ψ_t + δ_t, 0)), with c_i = 1, and c_t = 0, δ_t = 0 off the entries.
 * The bound on S: let a_t = Ψ_t + δ_t (δ_t = 0 off the entries), so S = Σ_t c_t·a_t − Σ_k c_k·δ_k.
 * With pg_t = a_t off the bound, ν_t·|a_t| <= rtol·V; so g(ν) − (S + Σ c_k·δ_k) = Σ_t (ν_t − c_t)·a_t
 * and each free token adds at most (ν_t − c_t)·|a_t| <= rtol·V, each token on its bound at most
 * (lo_t − c_t)·max(a_t, 0).  Trading nothing is feasible with S = 0, so the dual optimum (g minus the
 * constant) is >= 0, and S >= 0 − |T|·rtol·V − the box terms.  A filled row never pays more than its
 * limits by more than that certified gap (up to the rounding of fp64 sums).  The accuracy is relative
 * to the order's value V, not to the amount filled: a tiny partial fill is accurate only to rtol·V.
 * Outputs (cfmm_limit_out; every pointer may be NULL): those of cfmm_basket_out, plus surplus [q],
 * computed on the host in entry order from the first term received, each term a multiply c_k·paid_k
 * then a subtract (no fma).  A row that does not fill reads 0.  Ask a quote with
 * tok_cap = leg_cap = 0 for the sizes first.
 * cfmm_quote_limit_orders prices every row on the current state on its own; no state changes.
 * cfmm_execute_limit_orders runs the rows in batch order, each re-solved on the state the earlier
 * filled rows left; min_received (NULL: none; finite and >= 0) is the minimum received of i: an equal
 * value fills, a smaller one reverts with CFMM_ORDER_LIMIT.  The transition, bookkeeping, conflict
 * rule ({i} ∪ entries ∪ B) and levels are those of basket rows.
 * Single GPU.  Synchronous.  Before cfmm_finalize: CFMM_ERR_STATE.  q == 0 does nothing.
 * Errors: CFMM_ERR_INVALID before anything runs for the basket calls' argument errors, a null
 * limit_price, and a limit price that is NaN, Inf or negative. */
typedef struct {
  double *paid;                                  /* [basket_off[q]] */
  double *received;                              /* [q] */
  uint8_t *status;                               /* [q] */
  int *solver_status, *iterations, *fun_evals;   /* [q] */
  double *merit;                                 /* [q] */
  int64_t *tok_off;                              /* [q+1] */
  int64_t tok_cap;
  int64_t *token;                                /* [tok_off[q]] */
  double *nu, *psi;                              /* [tok_off[q]] */
  int64_t *leg_off;                              /* [q+1] */
  int64_t leg_cap;
  int *leg_type;                                 /* [leg_off[q]] */
  int64_t *leg_pool;                             /* [leg_off[q]] */
  double *leg_delta, *leg_lambda;                /* [2·leg_off[q]] */
  double *surplus;                               /* [q] */
} cfmm_limit_out;
int cfmm_quote_limit_orders(cfmm_ctx *ctx, int64_t q, const int64_t *token_out /* [q] */,
                            const int64_t *basket_off /* [q+1] */,
                            const int64_t *basket_token /* [basket_off[q]] */,
                            const double *basket_amount /* [basket_off[q]] */,
                            const double *limit_price /* [basket_off[q]] */,
                            const uint8_t *allowed /* [n_tokens], required */,
                            const cfmm_subgraph_opts *opts /* NULL = defaults */, cfmm_limit_out *out);
int cfmm_execute_limit_orders(cfmm_ctx *ctx, int64_t q, const int64_t *token_out,
                              const int64_t *basket_off, const int64_t *basket_token,
                              const double *basket_amount, const double *limit_price,
                              const double *min_received /* [q] or NULL */, const uint8_t *allowed,
                              const cfmm_subgraph_opts *opts, cfmm_limit_out *out);

/* ---- per-row masks: each subgraph, basket and limit row over its own allowed tokens -----------
 * cfmm_{quote,execute}_subgraph_swap_orders_rows, cfmm_{quote,execute}_basket_swap_orders_rows and
 * cfmm_{quote,execute}_limit_orders_rows take the arguments of the calls without _rows, with one
 * difference: in place of the mask `allowed` they take a per-row CSR
 *   allow_off [q+1], allow_token [allow_off[q]] (1-based),
 * and row r's allowed tokens are allow_token[allow_off[r] .. allow_off[r+1]), in any order.  The list
 * may be empty and may hold the row's own tokens (j and i; for baskets and limits i and the entries).
 * Row r is defined exactly as the call without _rows with `allowed` = row r's list: B_r is the list
 * minus the row's own tokens, and T, the component rule, the pool list in global insertion order, the
 * local token order (…, then B_r ∩ T ascending), the dual, box, start, optimizer, stop, the fill
 * promises, the outputs and the execute transition are that call's.  A row's bits depend on its own
 * tokens and list alone, not on the batch or on the other rows' lists.  What differs:
 *   size     at most CFMM_SUBGRAPH_MAX_TOKENS tokens in B_r (subgraph rows); basket and limit rows keep
 *            the basket calls' limit on basket ∪ B_r (CFMM_SUBGRAPH_MAX_TOKENS + 1 tokens besides i).
 *   work     each row's CTA builds its row's slot graph (the list sorted, the pairs among its tokens and
 *            their activity) before its setup.  The device workspace adds b² · 7 bytes per resident
 *            CTA, b the call's longest list (at most CFMM_SUBGRAPH_MAX_TOKENS + 2 tokens: about 466 KB
 *            per CTA), and the grid stays one wave of resident CTAs, as without _rows.
 *   execute  two rows conflict when their own token sets {j, i} ∪ B_r (baskets and limits:
 *            {i} ∪ entries ∪ B_r) intersect; rows are leveled by cfmm_execute_paths' rule over one
 *            n_tokens table, so rows on disjoint token sets share a level and its launches.
 * Errors: CFMM_ERR_INVALID before anything runs or changes for every error of the call without _rows
 * (its null-mask error aside), and for a null allow_off, a null allow_token when allow_off[q] > 0, an
 * allow_off that does not start at 0 or that decreases, a listed token outside 1..n_tokens, a token
 * listed twice in one row, and a row over the size limit.  Single GPU. */
int cfmm_quote_subgraph_swap_orders_rows(cfmm_ctx *ctx, int64_t q, const int64_t *token_in /* [q] */,
                                         const int64_t *token_out /* [q] */,
                                         const uint8_t *kind /* [q] or NULL: all exact-in */,
                                         const double *amount /* [q] */, const int64_t *allow_off /* [q+1] */,
                                         const int64_t *allow_token /* [allow_off[q]] */,
                                         const cfmm_subgraph_opts *opts /* NULL = defaults */,
                                         cfmm_subgraph_out *out);
int cfmm_execute_subgraph_swap_orders_rows(cfmm_ctx *ctx, int64_t q, const int64_t *token_in,
                                           const int64_t *token_out, const uint8_t *kind,
                                           const double *amount, const double *limit /* [q] or NULL */,
                                           const int64_t *allow_off, const int64_t *allow_token,
                                           const cfmm_subgraph_opts *opts, cfmm_subgraph_out *out);
int cfmm_quote_basket_swap_orders_rows(cfmm_ctx *ctx, int64_t q, const int64_t *token_out /* [q] */,
                                       const int64_t *basket_off /* [q+1] */,
                                       const int64_t *basket_token /* [basket_off[q]] */,
                                       const uint8_t *entry_kind /* [basket_off[q]] or NULL: every entry sold */,
                                       const double *basket_amount /* [basket_off[q]] */,
                                       const int64_t *allow_off /* [q+1] */,
                                       const int64_t *allow_token /* [allow_off[q]] */,
                                       const cfmm_subgraph_opts *opts /* NULL = defaults */,
                                       cfmm_basket_out *out);
int cfmm_execute_basket_swap_orders_rows(cfmm_ctx *ctx, int64_t q, const int64_t *token_out,
                                         const int64_t *basket_off, const int64_t *basket_token,
                                         const uint8_t *entry_kind, const double *basket_amount,
                                         const double *limit /* [q] or NULL */, const int64_t *allow_off,
                                         const int64_t *allow_token, const cfmm_subgraph_opts *opts,
                                         cfmm_basket_out *out);
int cfmm_quote_limit_orders_rows(cfmm_ctx *ctx, int64_t q, const int64_t *token_out /* [q] */,
                                 const int64_t *basket_off /* [q+1] */,
                                 const int64_t *basket_token /* [basket_off[q]] */,
                                 const double *basket_amount /* [basket_off[q]] */,
                                 const double *limit_price /* [basket_off[q]] */,
                                 const int64_t *allow_off /* [q+1] */, const int64_t *allow_token /* [allow_off[q]] */,
                                 const cfmm_subgraph_opts *opts /* NULL = defaults */, cfmm_limit_out *out);
int cfmm_execute_limit_orders_rows(cfmm_ctx *ctx, int64_t q, const int64_t *token_out,
                                   const int64_t *basket_off, const int64_t *basket_token,
                                   const double *basket_amount, const double *limit_price,
                                   const double *min_received /* [q] or NULL */, const int64_t *allow_off,
                                   const int64_t *allow_token, const cfmm_subgraph_opts *opts,
                                   cfmm_limit_out *out);

/* ---- arbitrage against external prices over every pool among allowed tokens ----------------
 * A row values tokens at external prices c and trades through every pool among its priced tokens to
 * maximise cᵀΨ with no token's net flow negative: route! with LinearNonnegative(c)
 * (src/objectives.jl:51-79) restricted to the row's pools, one convex dual per row.
 *   A        the tokens t with allowed[t-1] != 0 (allowed [n_tokens], required; one mask per call),
 *            ascending; n_A <= CFMM_PRICE_ARB_MAX_TOKENS.
 *   price    [q·n_A], row-major, columns in A's order.  Each price is 0 (the token is not in this
 *            row) or finite and > 0, and every row has a positive price.
 *   T        the row's priced tokens that hold at least one active pool whose two tokens are both
 *            priced.  Every component of T is an arbitrage of its own; every token in it has a price.
 *   pools    every pool of every pair inside T, all three types, appended pools included, retired
 *            pools listed (they trade (0, 0)), in global insertion order, as for subgraph orders.
 *   tokens   local order: T ascending.
 * Problem.  Minimise g(ν) = Σ_p π_p(ν) on the box ν_t >= c_t + 1e-8 (one IEEE addition, as
 * LinearNonnegative's lower limit), with no upper bound and no linear term.  Legs, the Ψ sums and the
 * value sum are those of subgraph orders, bit for bit in their operation order; the gradient is Ψ.
 *   start    ν⁰ = the box's lower bound: the caller's prices are the point the arbitrage is measured
 *            from (no breadth-first pricing).
 *   stop     m_r = max_t ν_t·|pg_t| / g(ν) at the committed iterate (g: the committed dual value,
 *            its profit: π is positively homogeneous, so g = νᵀΨ).  Status 0 when m_r <= rtol; the
 *            other statuses as cfmm_solve.  mx = max_t ν_t·|pg_t| = 0 gives m_r = 0; mx > 0 with
 *            g <= 0 gives m_r = +inf.  A row where no pool trades at ν⁰ (T empty included) fills with
 *            zeros after that one evaluation: solver status 0, 0 iterations, 1 evaluation, m_r = 0.
 * What a fill promises.  A row fills only at solver status 0 (else CFMM_ORDER_NOT_CONVERGED, with
 * zero legs and profit; ν, Ψ and m_r stay those of the last iterate).  A filled row has
 * profit = Σ_t c_t·Ψ_t in local order (the first term alone, then IEEE additions), and, from
 * m_r <= rtol with ν_t·|pg_t| <= rtol·g:
 *   each token's net Ψ_t >= −rtol·g/ν_t (the caller funds at most that much of t);
 *   g − cᵀΨ = Σ_t (ν_t − c_t)·Ψ_t <= |T|·rtol·g + Σ_{t on its bound} 1e-8·max(Ψ_t, 0), each free
 *   token adding at most (ν_t − c_t)·rtol·g/ν_t <= rtol·g, so the duality gap against the optimum
 *   (at most g) is at most |T|·rtol·g plus the box terms (up to the rounding of fp64 sums).
 * Outputs (cfmm_price_arb_out; every pointer may be NULL): per row profit, status (CFMM_ORDER_*),
 * solver_status, iterations, fun_evals, merit (m_r); tokens and legs as cfmm_subgraph_out.  Ask a
 * quote with tok_cap = leg_cap = 0 for the sizes first.
 * cfmm_quote_price_arbitrage prices every row on the current state on its own; no state changes.
 * cfmm_execute_price_arbitrage runs the rows in batch order, each re-solved on the state the earlier
 * filled rows left.  min_profit (NULL: none; finite and >= 0) is the minimum profit: an equal profit
 * fills, a smaller one reverts with CFMM_ORDER_LIMIT.  A filled row applies split_leg's transition at
 * its ν, then the bookkeeping of cfmm_execute_swaps.  Two rows conflict when their priced tokens
 * overlap (a row's T lies in them); rows are leveled by cfmm_execute_paths' rule, one launch per
 * level, so rows on disjoint price subsets share a launch.  An execute whose token or leg outputs are
 * given with a cap below the size is rejected before anything changes.
 * Options: cfmm_subgraph_opts, with its defaults.  Single GPU.  Synchronous.  Before cfmm_finalize:
 * CFMM_ERR_STATE.  q == 0 does nothing.  CFMM_ERR_INVALID before anything runs for: q < 0; a null
 * price or allowed; more than CFMM_PRICE_ARB_MAX_TOKENS allowed tokens; a price that is negative,
 * NaN or Inf; a row with no positive price; the option errors of subgraph orders; a min_profit that
 * is NaN, negative or Inf. */
#define CFMM_PRICE_ARB_MAX_TOKENS (CFMM_SUBGRAPH_MAX_TOKENS + 2)
typedef struct {
  double *profit;                                /* [q] */
  uint8_t *status;                               /* [q] */
  int *solver_status, *iterations, *fun_evals;   /* [q] */
  double *merit;                                 /* [q] */
  int64_t *tok_off;                              /* [q+1] */
  int64_t tok_cap;
  int64_t *token;                                /* [tok_off[q]] */
  double *nu, *psi;                              /* [tok_off[q]] */
  int64_t *leg_off;                              /* [q+1] */
  int64_t leg_cap;
  int *leg_type;                                 /* [leg_off[q]] */
  int64_t *leg_pool;                             /* [leg_off[q]] */
  double *leg_delta, *leg_lambda;                /* [2·leg_off[q]] */
} cfmm_price_arb_out;
int cfmm_quote_price_arbitrage(cfmm_ctx *ctx, int64_t q, const double *price /* [q·n_A] */,
                               const uint8_t *allowed /* [n_tokens], required */,
                               const cfmm_subgraph_opts *opts /* NULL = defaults */,
                               cfmm_price_arb_out *out);
int cfmm_execute_price_arbitrage(cfmm_ctx *ctx, int64_t q, const double *price,
                                 const double *min_profit /* [q] or NULL */, const uint8_t *allowed,
                                 const cfmm_subgraph_opts *opts, cfmm_price_arb_out *out);

/* ---- arbitrage against external prices from inventory: one token list per row, with holdings ----
 * A row values its own tokens at external prices c and trades through every pool among them to
 * maximise cᵀΨ, where the net may spend up to what the caller holds: route! with the objective
 * cᵀΨ − I(Ψ + h >= 0) restricted to the row's pools.  h = 0 is LinearNonnegative(c); c = e_i with
 * h = Δin is BasketLiquidation(i, Δin); c = 1 at i and limit_k at each sold k is LimitBasket.
 *   L_r      the row's tokens allow_token[allow_off[r] .. allow_off[r+1]) (1-based, distinct, any
 *            order, 1 to CFMM_PRICE_ARB_MAX_TOKENS of them).
 *   price    aligned with allow_token: c_t finite and >= 0, and every row has a c_t > 0.  A token
 *            priced 0 stays in the row as an intermediate valued at 0 (unlike the one-mask call).
 *   holding  aligned with allow_token, or NULL (every h_t = 0): h_t finite and >= 0.
 *   T        the listed tokens that hold an active pool to another listed token.
 *   pools    every pool of every pair inside T, as the one-mask call (global insertion order,
 *            retired pools listed); local token order T ascending.
 * Problem.  Minimise G(ν) = Σ_p π_p(ν) + hᵀν on the box ν_t >= c_t + 1e-8 (one IEEE addition), with
 * no upper bound; the linear term is h, and hᵀν is summed over the held tokens in a fixed order (the
 * CTA sum's tree over them in local order).  P̄ = G − hᵀc = π(ν) + hᵀ(ν − c) >= 0 on the box bounds
 * the profit from above.
 *   start    the box's lower bound, as the one-mask call.
 *   stop     mx = max_t s_t·|pg_t| with s_t = max(ν_t, c̄), c̄ the least positive price the row lists,
 *            and m_r = mx / P̄ at the committed iterate (0 when mx = 0, +inf when P̄ <= 0 < mx).
 *            Status 0 when m_r <= rtol or mx <= atol (atol in the price unit, default 0); the other
 *            statuses as cfmm_solve.  A priced token has ν_t > c_t >= c̄, so s_t = ν_t there; the floor
 *            c̄ keeps a price-0 token, which sits near ν_t = 1e-8, measured in token units.  atol > 0
 *            lets a row with nothing worth doing stop at once instead of running to max_iter as g goes
 *            to 0 with mx.
 * What a fill promises (ε = max(rtol·P̄, atol); derived in price_arb_kernels.cuh):
 *   Ψ_t >= −h_t − ε/max(ν_t, c̄) for every token: the row spends at most its holding, up to ε/c̄ units
 *   of any token;
 *   profit = Σ_t c_t·Ψ_t in local order (the first term alone, then IEEE additions);
 *   P̄ − cᵀΨ = Σ_t (ν_t − c_t)(Ψ_t + h_t) <= |T|·ε + Σ_{t on its bound} 1e-8·(Ψ_t + h_t).  P̄ bounds
 *   the optimum profit from above; cᵀΨ exceeds P̄ by at most the overdraft valued at ν,
 *   Σ_t (ν_t − c_t)·max(−Ψ_t − h_t, 0) <= |T|·ε (up to the rounding of fp64 sums).
 * A row with no holding, atol 0 and every listed price > 0 runs the one-mask call's operations (lin 0,
 * linear value 0.0, s_t = ν_t, m_r = mx / g): its outputs equal cfmm_quote_price_arbitrage's with its list as the
 * mask and its prices, bit for bit.
 * Outputs: cfmm_price_arb_out, as the one-mask call (a row fills only at solver status 0).
 * cfmm_quote_price_arbitrage_rows prices every row on the current state on its own; no state changes.
 * cfmm_execute_price_arbitrage_rows runs the rows in batch order, each re-solved on the state the
 * earlier filled rows left; min_profit (NULL: none; finite and >= 0) reverts a row below it with
 * CFMM_ORDER_LIMIT (an equal profit fills).  Two rows conflict when their lists intersect; rows are
 * leveled by cfmm_execute_paths' rule, so rows on disjoint lists share a level and its launch.  An
 * execute whose token or leg outputs are given with a cap below the size is rejected before anything
 * changes.  Each row's CTA builds its slot graph as the _rows order calls do (b² · 7 bytes of device
 * workspace per resident CTA, b the longest list).
 * Options: cfmm_price_arb_opts (NULL: cfmm_subgraph_opts' defaults and atol 0).  Single GPU.
 * Synchronous.  Before cfmm_finalize: CFMM_ERR_STATE.  q == 0 does nothing.  CFMM_ERR_INVALID before
 * anything runs for: q < 0; a null allow_off, a null allow_token when allow_off[q] > 0, a null price;
 * an allow_off that does not start at 0 or that decreases; a list that is empty or longer than
 * CFMM_PRICE_ARB_MAX_TOKENS; a token outside 1..n_tokens or listed twice in a row; a price or holding
 * that is negative, NaN or Inf; a row with no positive price; the option errors of subgraph orders;
 * an atol that is not finite or is < 0; a min_profit that is NaN, negative or Inf. */
typedef struct {
  int max_iter, max_fun;
  double rtol, factr;
  double atol; /* the absolute stop on max_t ν_t·|pg_t|, >= 0 */
} cfmm_price_arb_opts;
int cfmm_quote_price_arbitrage_rows(cfmm_ctx *ctx, int64_t q, const int64_t *allow_off /* [q+1] */,
                                    const int64_t *allow_token /* [allow_off[q]] */,
                                    const double *price /* [allow_off[q]] */,
                                    const double *holding /* [allow_off[q]] or NULL */,
                                    const cfmm_price_arb_opts *opts /* NULL = defaults */,
                                    cfmm_price_arb_out *out);
int cfmm_execute_price_arbitrage_rows(cfmm_ctx *ctx, int64_t q, const int64_t *allow_off,
                                      const int64_t *allow_token, const double *price, const double *holding,
                                      const double *min_profit /* [q] or NULL */,
                                      const cfmm_price_arb_opts *opts, cfmm_price_arb_out *out);

/* ---- UniV3 liquidity changes: mint and burn price ranges ---------------------------------
 * A UniV3 pool's ladder is T₁ > T₂ > … > Tₙ (lower_ticks); tick i holds liquidity Lᵢ on the
 * prices (Tᵢ₊₁, Tᵢ], the last tick Lₙ on (0, Tₙ] (tick_high_price / tick_low_price,
 * src/cfmms.jl:251-259).  A row (pool, lo, hi, dL) needs 0 < lo < hi, both finite, and dL finite
 * and != 0 (dL > 0 mints, dL < 0 burns).  The rows are applied in batch order, with the result of
 * applying them one at a time:
 *   boundaries  hi and lo are inserted unless some Tᵢ equals them bit for bit.  A boundary inside
 *               tick i splits it; both parts carry Lᵢ (copied).  A boundary above T₁ adds a new
 *               first tick (T₁, b] with liquidity 0 (b is the new T₁); one below Tₙ splits the
 *               last tick.
 *   liquidity   every tick whose upper bound Tᵢ satisfies lo < Tᵢ <= hi gets Lᵢ <- Lᵢ + dL, one
 *               IEEE addition (round to nearest), in batch order per tick.
 *   rejection   a row that leaves a tick it added to with L < 0 or L not finite rejects the whole
 *               call with CFMM_ERR_INVALID; the message names the first such row, and no pool
 *               changes.  Burning exactly x from a tick that an earlier mint of x raised from
 *               L >= 0, with only mints on that tick in between, never fails: rounding is
 *               monotonic, so the tick holds at least x and the difference is >= 0.
 *   unchanged   the current price q.  current_tick is re-derived (searchsortedlast, :235) and
 *               every tick's compute_at_tick record rebuilt on the device.  Boundaries are never
 *               removed: a range burned to zero stays as an empty tick, which walks pass through.
 * Retired pools (cfmm_set_active) take the change in the state they keep; their records stay
 * empty until they are restored.  Afterwards the state version moves (captured sweep graphs
 * re-capture; the tick arrays may have been reallocated), the materialised trades stay (as after
 * cfmm_execute_swaps), cfmm_apply_trades clamps to the current T₁, cfmm_update_univ3 validates
 * prices against the current T₁ and takes liquidity in the current CSR order.
 *
 * Before cfmm_finalize: CFMM_ERR_STATE.  A pool outside the UniV3 pools, a NaN or Inf, lo <= 0,
 * lo >= hi or dL == 0: CFMM_ERR_INVALID before anything runs.  q == 0 does nothing.  A call that
 * would take a main or appended set past 2^31-1 ticks is rejected (CFMM_ERR_INVALID) before
 * anything changes; CFMM_ERR_NOMEM if the grown tick arrays cannot be allocated, with no pool
 * changed. */
/* q rows on UniV3 pools; pool: [q] UniV3 insertion order (tails included);
 * range: [2q] pool-major (lo, hi); dL: [q].  Synchronous. */
int cfmm_modify_univ3_liquidity(cfmm_ctx *ctx, int64_t q, const int64_t *pool,
                                const double *range, const double *dL);
/* The current ladders of UniV3 pools [first, first+count): tick_off [count+1] always;
 * lower_ticks / liquidity (may be NULL) [tick_off[count]].  Retired pools report their kept state. */
int cfmm_get_univ3_ticks(cfmm_ctx *ctx, int64_t first, int64_t count, int64_t *tick_off,
                         double *lower_ticks, double *liquidity);

/* ---- the outer iteration on the device (SURVEY §8f rank 2) ---------------------------
 * Minimises the dual g(nu) = lin' nu + sum_i arb_i(nu) over the box lower <= nu <= upper
 * -- route! (src/router.jl:58-108) for objectives of the form f(nu) = lin' nu on a box,
 * which both objectives of the reference are (src/objectives.jl:62-79: lin = 0, lower =
 * c + 1e-8; :106-129: lin = Delta_in with lin[i] = 0, lower = sqrt(eps), 1 + sqrt(eps) at
 * i).  nu, the gradient, the L-BFGS history (m = 5) and the search direction stay in device
 * memory; every function/gradient evaluation is one sweep plus vector kernels, and only a
 * few scalars cross PCIe per evaluation.  The optimizer is a projected L-BFGS with Armijo
 * backtracking, not the Fortran L-BFGS-B: same minimiser of the convex dual, different
 * iterates.  On return v_out holds the final nu and the trades at it are materialised
 * (cfmm_get_trades), as after route!.  lin and upper may be NULL (0 / +inf), v0 NULL =
 * ones/n (router.jl:62).  status: 0 projected gradient <= pgtol, 1 relative decrease <=
 * factr*eps or no further move, 2 max_iter, 3 max_fun, 4 line search failed, 5 NaN. */
typedef struct {
  int max_iter, max_fun;
  double pgtol, factr;
} cfmm_solve_opts;
typedef struct {
  int iterations, fun_evals, status;
  double f, pg_norm, solve_ms;
} cfmm_solve_info;
int cfmm_solve(cfmm_ctx *ctx, const double *lin, const double *lower, const double *upper,
               const double *v0, const cfmm_solve_opts *opts /* NULL = route!'s defaults */,
               double *v_out, cfmm_solve_info *info /* may be NULL */);

/* Tunables (none is needed for normal use).
 *   "exact"            1 = evaluate all four closed forms exactly as written in the
 *                      reference for every pool; 0 (default) = evaluate only the side that
 *                      can trade, falling back to the full form near ties (same bits).
 *   "gradient_math"    gradient-only sweeps, where per-pool trades are not observable:
 *                      1 (default) = economized closed forms (ProductTwoCoin: one rsqrt +
 *                      one rcp; GeometricMean: one pow), <= ~3 ulp of the reserve per pool;
 *                      0 = the reference's operation order, bit-identical per pool.
 *                      Materialising sweeps and "exact" are always bit-identical.
 *   "tma_variant"      0 (default) = b-bucketed ProductTwoCoin layout + TMA kernel for
 *                      gradient-only sweeps; -1 = token-sorted layout, first-generation
 *                      kernel only.  Fixes the pool layout: before cfmm_finalize.
 *   "psi_fixed_point"  Ψ[b] partial sums of the TMA kernel: 1 (default) = 64-bit fixed
 *                      point on native 32-bit shared atomics (quantum <= 2^-59 of the
 *                      token's total reserve; used when every token's pools span <= 2^40
 *                      in reserve and totals lie within 2^+-200), 0 = fp64 CAS adds.
 *   "orient_by_degree" store each ProductTwoCoin pool with its higher-degree token first:
 *                      -1 (default) = only when finalize detects hub tokens, 0 never,
 *                      1 always; before cfmm_finalize.
 *   "use_tma"          0 = run the first-generation kernel on the same layout.
 *   "blocks_per_sm"    resident CTAs per SM of the persistent kernels (measurement knob).
 *   "grid_waves"       sweep_kernel (UniV3, materialising sweeps): 1 (default) = one wave of
 *                      resident CTAs striding over the pools, 0 = one CTA per 512 pools (hardware
 *                      block scheduling), N = N waves (measurement knob).
 *   "fused_exchange"   multi-GPU: 1 (default) = product-only sweeps run the peer exchange
 *                      in the sweep kernel's tail; 0 = separate exchange launch.
 *   "coop_launch"      multi-GPU: 1 = the fused sweep+exchange kernel is launched with
 *                      cudaLaunchCooperativeKernel (the driver guarantees that every CTA of its
 *                      grid barrier is resident, or fails the launch); 0 (default) = plain launch,
 *                      residency follows from the occupancy query that sizes the persistent grid,
 *                      and a barrier that cannot complete ends in CFMM_ERR_COMM after the poll
 *                      bound instead of hanging.
 *   "exchange_bypass"  multi-GPU: 1 = sweeps skip the exchange and return this rank's partial
 *                      [psi ; acc] (verification; every rank must set it alike).
 *   "exchange_protocol" multi-GPU: how [psi ; acc] is summed over NVLink peer memory: 3 = direct
 *                      push, one hop, 8 bytes per value (a receive slot is "empty" or a value);
 *                      1 = LL one-shot (16-byte epoch-tagged packets, one hop); 2 = LL two-shot
 *                      (reduce-scatter + all-gather, two hops, fewest bytes); 0 (default) = by
 *                      group size: 3 up to 4 ranks, 2 beyond.  Every rank of the group must use
 *                      the same one.
 *   "exchange_two_shot" multi-GPU: 0 / 1 = "exchange_protocol" 1 / 2.
 *   "sweep_events"     1 = record the two CUDA events cfmm_last_sweep_ms needs around every
 *                      sweep (default 0; turns the sweep graphs off).
 *   "sweep_graphs"     1 (default) = cfmm_sweep replays {H2D nu, sweep, D2H [psi; acc]} as one
 *                      CUDA graph once the same pinned host buffers (cfmm_host_alloc, psi and
 *                      acc contiguous) have been passed twice with unchanged options.
 *   "geomean_log2"     gradient-only GeometricMean sweeps take the power as exp2(e*log2 t)
 *                      (1, default; <= 12 ulp over the admitted range, validated against
 *                      pow on hardware) or as pow (0).
 *   "compact_stream"   1 (default) = economized ProductTwoCoin sweeps stream 20-byte pool records
 *                      (fee through a dictionary of <= 256 distinct values, first token relative
 *                      to its record's first, second token relative to its bucket) when the
 *                      pool set allows it (<= 256 fees, the first tokens of every pair of
 *                      consecutive 96-pool chunks of a bucket spanning < 8192);
 *                      0 = 32-byte records.
 *   "compact_record"   pools per record of that stream: 192 (two chunks of a bucket, one bulk
 *                      copy, six pools per thread), 96, or 0 (default) = 192 when the set has at
 *                      least 4 such records per resident warp, else 96.
 *   "l2_keep"          gradient sweeps that stream 192-pool records ("compact_record") larger in
 *                      all than the device's L2:
 *                      the bulk copies carry L2 eviction hints: the first h records of every
 *                      CTA's range as evict_last, every other record as evict_first, so that the
 *                      records each sweep waits for at its start stay in the L2 from one sweep
 *                      to the next and come from there instead of HBM.  -1 (default) = h chosen
 *                      from the L2 size (two records per warp of a CTA, the kept records taking
 *                      at most 40 % of the L2), 0 = no hints, h > 0 = that h.  Streams that fit
 *                      in the L2 run without hints whatever the value.  Only per-instruction
 *                      hints: no L2 set-aside, no access-policy window; the kept lines go back
 *                      to evict_normal when the rule or the stream changes and at cfmm_destroy.
 *                      Results do not depend on it.
 *   "geomean_tma"      1 (default) = gradient-only GeometricMeanTwoCoin sweeps run on the TMA
 *                      kernel too (48-byte records, same fixed-point slice); 0 = first-generation
 *                      kernel.
 *   "balance"          TMA kernel: 1 (default) = every CTA's chunk range is sized by its measured
 *                      speed (durations are fed back through device memory and an occasional
 *                      asynchronous copy, and the range table is re-derived between launches);
 *                      0 = even split.
 *   "trace"            1 = TMA sweeps record per-CTA phase timestamps (cfmm_debug_read_trace).
 *   "profile"          N = time the next N kernel launches (cfmm_profile_read). */
int cfmm_set_option(cfmm_ctx *ctx, const char *key, int64_t value);

/* Device time (ms, CUDA events on the sweep stream) of the kernels of the
 * last cfmm_sweep / cfmm_sweep_device call; synchronises the stream. */
int cfmm_last_sweep_ms(cfmm_ctx *ctx, float *ms_out);
/* Number of kernel launches issued by this context so far. */
int64_t cfmm_launch_count(const cfmm_ctx *ctx);

/* Per-kernel device timing.  cfmm_set_option(ctx, "profile", N) arms CUDA-event
 * pairs for the next N kernel launches (recorded on the launching stream,
 * around each sweep kernel / the peer exchange).  cfmm_profile_read sums the
 * durations recorded so far for one pool type (cfmm_pool_type, 3 = the multi-GPU
 * exchange kernel, or 4 = the kernels of cfmm_quote_swaps / cfmm_execute_swaps /
 * cfmm_quote_swaps_exact_out / cfmm_execute_swap_orders / cfmm_quote_paths /
 * cfmm_execute_paths / cfmm_pair_pools / cfmm_quote_split_orders /
 * cfmm_execute_split_orders / cfmm_quote_routed_orders / cfmm_execute_routed_orders /
 * cfmm_choose_order_hubs / cfmm_find_order_paths / cfmm_quote_token_values, the pair-index
 * build counted as one launch); it
 * synchronises on the recorded events.
 * cfmm_profile_reset re-arms the same N pairs. */
int cfmm_profile_read(cfmm_ctx *ctx, int type, double *total_ms, int64_t *launches);
/* The individual durations (ms) behind cfmm_profile_read, in launch order: fills
 * ms_out[0 .. min(cap, *n_out)) and sets *n_out to the number recorded for `type`. */
int cfmm_profile_read_times(cfmm_ctx *ctx, int type, float *ms_out, int64_t cap, int64_t *n_out);
int cfmm_profile_reset(cfmm_ctx *ctx);

/* Test hook: counts, over n operand pairs (host arrays), the results of the
 * kernels' guard-free in-range division / square root that differ from IEEE
 * a/b, sqrt(a), sqrt(b).  0 for operands in [2^-100, 2^100]. */
int cfmm_selftest_inrange_math(cfmm_ctx *ctx, const double *a, const double *b,
                               int64_t n, int64_t *mismatches);

/* Test hook, needs no device: the layout cfmm_finalize would give m ProductTwoCoin
 * pools (Ai 1-based [2m]) for "tma_variant" `variant` and orientation mode `orient`.
 * info[6] = {m_padded, bucket width, bucketed?, hubs detected?, chunk size, variant};
 * with cap >= m_padded also order_out [m_padded] (device position -> pool index, -1 =
 * padding), chunk_bucket_out [m_padded / chunk] and swapped_out [m]. */
int cfmm_debug_product_layout(int64_t n_tokens, int64_t m, const int64_t *Ai, int orient,
                              int variant, int64_t cap, int64_t *order_out,
                              int32_t *chunk_bucket_out, uint8_t *swapped_out, int64_t *info);
/* Test hook: info[8] = {main-set pools, appended (tail) pools, main-set padded length, TMA
 * layout built, fixed-point psi slice allowed, compact stream allowed, every reserve in the
 * guard-free range, retired pools} of one pool type. */
int cfmm_debug_pool_set_info(cfmm_ctx *ctx, int type, int64_t *info);
/* Test hook: pools per compact record the next gradient-only sweep of the main set of
 * `type` streams under the current options: 192 (18-byte pool records), 96 (20-byte
 * pool records) or 0 (no compact stream: other pool types, exact or reference-order
 * math, or a set that does not fit it). */
int cfmm_debug_compact_record(cfmm_ctx *ctx, int type, int64_t *pools_per_record);
/* Test hook: the L2 keep rule (option "l2_keep") the next gradient-only sweep of the main
 * ProductTwoCoin set runs with: h > 0 = the first h records of every CTA's range are kept in the
 * L2 across sweeps, 0 = no L2 hints (other pool types, a stream other than the 192-pool records, a stream
 * that fits in the L2, or l2_keep = 0). */
int cfmm_debug_l2_keep(cfmm_ctx *ctx, int type, int64_t *keep);
/* Measurement hook (option "trace" = 1): per-CTA phase timestamps of the last TMA gradient
 * sweep, ns of %globaltimer: out[8 * grid] = {entry, price slice ready, own range done,
 * all chunks done, partials flushed, exit, grid barrier passed (fused exchange, else 0),
 * SM id << 32 | chunks processed} per CTA. */
int cfmm_debug_read_trace(cfmm_ctx *ctx, uint64_t *out, int64_t cap_ctas, int64_t *grid_out);

/* ---- pinned host memory helpers ------------------------------------------- */
void *cfmm_host_alloc(size_t bytes);
void cfmm_host_free(void *p);

/* ---- multi-GPU: one context per GPU, one process per GPU ------------------ */
/* Pools shard across ranks (each rank adds only its shard); the only exchange
 * is the sum of [psi ; acc] (n_tokens+1 fp64) after each sweep.  The exchange
 * runs over NVLink peer memory: every rank exports a handle to its exchange
 * buffer, the host side all-gathers the handles (any transport; the Python
 * host uses torch.distributed), and each rank attaches the others'. */
#define CFMM_COMM_HANDLE_BYTES 128
int cfmm_comm_export(cfmm_ctx *ctx, void *handle_out /* CFMM_COMM_HANDLE_BYTES */);
int cfmm_comm_attach(cfmm_ctx *ctx, int world, int rank,
                     const void *handles /* world * CFMM_COMM_HANDLE_BYTES */);
int cfmm_comm_detach(cfmm_ctx *ctx);
/* After asynchronous sweeps (cfmm_sweep_device*): waits for the stream of the last sweep and
 * returns CFMM_ERR_COMM if any exchange so far hit its poll bound (a rank that never launched
 * the matching sweep, a dead peer); CFMM_OK otherwise and for contexts outside a group.
 * cfmm_sweep makes the same check itself. */
int cfmm_comm_check(cfmm_ctx *ctx);

#ifdef __cplusplus
}
#endif
#endif /* CFMM_B200_H */
