"""Launches, profile entries and rejection messages of the swap, path, order, arbitrage and liquidity
calls (include/cfmm_b200.h), pinned per call.

Each call's cfmm_launch_count delta and its delta of event-timed entries in profile slot 4
(cfmm_profile_read) are fixed numbers on one seeded context holding all three pool types, with
appended pools, retired pools and multi-tick UniV3 ladders: how a call's host code splits its work
into launches, and which of them it times, is part of what a caller measures.  The rejections pin the
exact code and message of the order calls' kind / amount / limit rules, and that each names the
first bad row."""
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

P, G, U = 0, 1, 2
N = 16  # tokens
PROF = 4  # cfmm_profile_read: the slot of the swap, path, order and arbitrage kernels
INVALID = -1  # CFMM_ERR_INVALID

# (launch_count delta, profile slot 4 entries delta) per call, in the order the calls run
EXPECTED = {
    "quote_swaps P": (2, 2),
    "quote_swaps G": (2, 2),
    "quote_swaps U": (2, 2),
    "quote_swaps_exact_out P": (2, 2),
    "quote_swaps_exact_out G": (2, 2),
    "quote_swaps_exact_out U": (2, 2),
    "execute_swaps P": (5, 2),
    "execute_swaps G": (5, 2),
    "execute_swaps U": (4, 2),
    "execute_swap_orders P": (5, 2),
    "execute_swap_orders G": (5, 2),
    "execute_swap_orders U": (4, 2),
    "execute_swap_orders U limits": (4, 2),
    "quote_paths": (2, 2),
    "execute_paths": (7, 2),
    "execute_paths levels": (9, 4),
    "pair_pools": (12, 4),
    "quote_split_orders": (2, 2),
    "execute_split_orders": (10, 2),
    "execute_split_orders limits legs": (11, 5),
    "quote_routed_orders": (5, 5),
    "execute_routed_orders levels": (10, 4),
    "quote_arbitrage": (2, 2),
    "execute_arbitrage": (8, 2),
    "scan_arbitrage": (16, 7),
    "modify_univ3_liquidity": (14, 0),
}


class Pools:
    """The seeded pool set: every type's pools in insertion order (main, then appended) with their
    token pairs, and the context."""

    def __init__(self, cr, synth):
        self.p = p = cr.DevicePools(N, device=0)
        Rp, gp, Ap = synth.product_pools(40, N, seed=11)
        Rg, gg, Ag, wg = synth.geomean_pools(20, N, seed=12)
        u = synth.univ3_pools(20, N, seed=13, ragged=True)
        p.add_product(Rp, gp, Ap)
        p.add_geomean(Rg, gg, Ag, wg)
        p.add_univ3(*u)
        p.finalize()
        Rp2, gp2, Ap2 = synth.product_pools(6, N, seed=21)
        Rg2, gg2, Ag2, wg2 = synth.geomean_pools(4, N, seed=22)
        u2 = synth.univ3_pools(4, N, seed=23, ragged=True)
        p.append_product(Rp2, gp2, Ap2)
        p.append_geomean(Rg2, gg2, Ag2, wg2)
        p.append_univ3(*u2)
        p.set_active(P, 3, [False])
        p.set_active(P, 41, [False])  # an appended pool
        p.set_active(U, 2, [False])
        self.Ai = {P: np.concatenate([Ap, Ap2]), G: np.concatenate([Ag, Ag2]), U: np.concatenate([u[2], u2[2]])}
        self.cp = np.concatenate([u[0], u2[0]])
        assert max(np.diff(u[3])) > 1 and max(np.diff(u2[3])) > 1  # multi-tick ladders in both UniV3 sets

    def pair(self, t, i):
        return [int(x) for x in self.Ai[t][i]]

    def next_hop(self, token, used):
        """A pool holding token that is not in used: (type, index, the token it passes on)."""
        for t in (U, P, G):
            for i, (a, b) in enumerate(self.Ai[t]):
                if (t, i) not in used and token in (a, b):
                    return t, i, int(b if a == token else a)
        raise AssertionError(f"no pool holds token {token}")

    def path(self, first, hops):
        """A path of `hops` hops from pool `first` (type, index), starting with its first token."""
        t, i = first
        start, token = self.pair(t, i)
        out, used = [(t, i)], {(t, i)}
        for _ in range(hops - 1):
            t, i, token = self.next_hop(token, used)
            out.append((t, i))
            used.add((t, i))
        return start, out

    def paths(self, specs):
        """CSR arrays of quote_paths for paths (first, hops, kind, amount)."""
        off, typ, pool, tok, kind, amount = [0], [], [], [], [], []
        for first, hops, k, a in specs:
            start, hs = self.path(first, hops)
            typ += [t for t, _ in hs]
            pool += [i for _, i in hs]
            off.append(len(typ))
            tok.append(start)
            kind.append(k)
            amount.append(a)
        return off, typ, pool, tok, kind, amount

    def unpaired(self):
        """A token pair no pool holds."""
        held = {tuple(sorted(self.pair(t, i))) for t in self.Ai for i in range(len(self.Ai[t]))}
        return next((a, b) for a in range(1, N + 1) for b in range(a + 1, N + 1) if (a, b) not in held)


@pytest.fixture(scope="module")
def pools(cr, synth):
    ps = Pools(cr, synth)
    yield ps
    ps.p.close()


def calls(ps):
    """(name, call) in the order they run; executes change the state the later calls see."""
    p = ps.p
    out = []
    tender = np.array([[1.0, 0.0], [0.0, 2.0], [0.5, 0.0], [0.0, 0.25], [3.0, 0.0]])
    want = np.array([[0.0, 1e-3], [1e-3, 0.0], [0.0, 2e-3], [1e-3, 0.0], [0.0, 1e-3]])
    rows = {P: [0, 3, 3, 7, 42], G: [1, 1, 5, 21, 23], U: [0, 2, 9, 9, 21]}  # main and appended, repeats
    for name, fn, arg in (("quote_swaps", p.quote_swaps, tender), ("quote_swaps_exact_out", p.quote_swaps_exact_out, want),
                          ("execute_swaps", p.execute_swaps, tender)):
        for t in (P, G, U):
            out.append((f"{name} {'PGU'[t]}", lambda fn=fn, t=t, arg=arg: fn(t, rows[t], arg)))
    kind = [0, 1, 0, 1, 0]
    amount = np.where(np.array(kind)[:, None] == 0, tender, want)
    for t in (P, G, U):
        out.append((f"execute_swap_orders {'PGU'[t]}",
                    lambda t=t: p.execute_swap_orders(t, rows[t], kind, amount)))
    out.append(("execute_swap_orders U limits",
                lambda: p.execute_swap_orders(U, rows[U], kind, amount, [0.0, math.inf, 1e300, 1.0, 0.0])))

    single = ps.paths([((P, 0), 3, 0, 0.5), ((U, 1), 2, 1, 1e-3), ((G, 22), 1, 0, 0.25)])
    out.append(("quote_paths", lambda: p.quote_paths(*single)))
    out.append(("execute_paths", lambda: p.execute_paths(*single)))
    shared = ps.paths([((P, 0), 2, 0, 0.5), ((P, 0), 1, 0, 0.25), ((U, 4), 3, 1, 1e-3), ((P, 0), 3, 0, 0.1)])
    out.append(("execute_paths levels", lambda: p.execute_paths(*shared, limit=[0.0, 0.0, 1e300, 0.0])))

    a0, b0 = ps.pair(P, 0)
    a1, b1 = ps.pair(U, 1)
    a2, b2 = ps.pair(G, 2)
    na, nb = ps.unpaired()
    tin, tout = [a0, a0, b1, na, a2, a0], [b0, b0, a1, nb, b2, b0]  # rows 0, 1, 5 share a pair
    skind, samount = [0, 1, 0, 0, 1, 0], [0.5, 1e-3, 0.25, 1.0, 1e-3, 0.1]
    out.append(("pair_pools", lambda: p.pair_pools(tin, tout)))
    out.append(("quote_split_orders", lambda: p.quote_split_orders(tin, tout, skind, samount)))
    out.append(("execute_split_orders", lambda: p.execute_split_orders(tin, tout, skind, samount)))
    out.append(("execute_split_orders limits legs",
                lambda: p.execute_split_orders(tin, tout, skind, samount, [0.0, 1e300, 0.0, 0.0, 1e300, 0.0],
                                               legs=True)))

    hubs = [h for h in range(1, N + 1) if h not in (a0, b0)][:3]
    hub_off = [0, 3, 3, 4, 6, 6]  # rows 0 and 3 route through the same hub pairs as row 2
    rt_in, rt_out = [a0, b1, a0, a0, na], [b0, a1, b0, b0, nb]
    rhubs = hubs + [hubs[0]] + [hubs[1], hubs[2]]
    rkind, ramount = [0, 1, 0, 1, 0], [0.5, 1e-3, 0.25, 1e-3, 1.0]
    out.append(("quote_routed_orders",
                lambda: p.quote_routed_orders(rt_in, rt_out, rkind, ramount, hub_off, rhubs, legs=True)))
    out.append(("execute_routed_orders levels",
                lambda: p.execute_routed_orders(rt_in, rt_out, rkind, ramount, hub_off, rhubs,
                                                [0.0, 1e300, 0.0, 1e300, 0.0])))

    base, other = [1, 1, 2], [3, 4, 5]
    ahub_off, ahubs = [0, 2, 2, 3], [6, 7, 8]
    out.append(("quote_arbitrage", lambda: p.quote_arbitrage(base, other, ahub_off, ahubs)))
    out.append(("execute_arbitrage", lambda: p.execute_arbitrage(base, other, ahub_off, ahubs, [0.0, 0.0, 1e-12])))

    def scan():
        found = p.scan_arbitrage([1, 2, 9], 1e-12, max_hubs=2, cap=64)[0]
        assert found > 0, "the scan found no rows"
    out.append(("scan_arbitrage", scan))

    lo = [ps.cp[1] * 0.9, ps.cp[21] * 0.5]  # pool 21 is an appended UniV3 pool
    hi = [ps.cp[1] * 1.1, ps.cp[21] * 3.0]
    out.append(("modify_univ3_liquidity", lambda: p.modify_univ3_liquidity([1, 21], lo, hi, [0.5, 0.25])))
    return out


def measure(ps):
    """{name: (launches, profile entries)} of every call, run in order."""
    p = ps.p
    p.set_option("profile", 4096)  # enough event slots for every call below
    got = {}
    for name, fn in calls(ps):
        l0, c0 = p.launch_count, p.profile_read(PROF)[1]
        fn()
        got[name] = (p.launch_count - l0, p.profile_read(PROF)[1] - c0)
    return got


def test_launches_and_profile_entries_per_call(pools):
    assert measure(pools) == EXPECTED


# ---- rejections: (code, message) of the first bad row ----------------------------------------

BAD = {  # name: (row 1's kind, amount, limit)
    "kind 2": (2, 1.0, 0.0),
    "amount nan": (0, math.nan, 0.0),
    "amount -1": (0, -1.0, 0.0),
    "amount +inf": (0, math.inf, 0.0),
    "limit nan": (0, 1.0, math.nan),
    "limit -1": (0, 1.0, -1.0),
    "exact-in +inf limit": (0, 1.0, math.inf),
}


def _expected_messages():
    """The messages of the four order calls, row 1 bad (row 0 is good)."""
    out = {}
    for call, noun in (("execute_swap_orders", "row"), ("execute_paths", "path"), ("execute_split_orders", "row"),
                       ("execute_routed_orders", "row")):
        for bad in BAD:
            if bad == "kind 2":
                msg = f"{call}: {noun} 1: kind 2 is neither exact-in (0) nor exact-out (1)"
            elif bad.startswith("amount"):
                amount = {"amount nan": "nan", "amount -1": "-1", "amount +inf": "inf"}[bad]
                msg = (f"{call}: row 1: tender ({amount}, 0) must be finite and >= 0" if call == "execute_swap_orders"
                       else f"{call}: {noun} 1: amount {amount} must be finite and >= 0")
            elif bad == "exact-in +inf limit":
                msg = f"{call}: {noun} 1: an exact-in {noun}'s minimum received must be finite"
            else:
                msg = f"{call}: {noun} 1: limit {'nan' if bad == 'limit nan' else '-1'} must be >= 0"
            out[(call, bad)] = msg
    return out


def rejections(ps):
    """{(call, bad input): (code, message)} of the four order calls."""
    import cfmmrouter_b200 as cr
    p = ps.p
    a0, b0 = ps.pair(P, 0)
    path = ps.paths([((P, 0), 2, 0, 0.5), ((P, 1), 1, 0, 0.5)])
    got = {}
    for bad, (k, a, l) in BAD.items():
        kind, amount, limit = [0, k], [0.5, a], [0.0, l]
        runs = {
            "execute_swap_orders": lambda: p.execute_swap_orders(P, [0, 1], kind, [[0.5, 0.0], [a, 0.0]], limit),
            "execute_paths": lambda: p.execute_paths(path[0], path[1], path[2], path[3], kind, amount, limit),
            "execute_split_orders": lambda: p.execute_split_orders([a0, a0], [b0, b0], kind, amount, limit),
            "execute_routed_orders": lambda: p.execute_routed_orders([a0, a0], [b0, b0], kind, amount, [0, 0, 0], [],
                                                                     limit),
        }
        for call, run in runs.items():
            with pytest.raises(cr.CFMMError) as e:
                run()
            got[(call, bad)] = (e.value.code, e.value.message)
    return got


def test_order_rejections(pools):
    expected = {key: (INVALID, msg) for key, msg in _expected_messages().items()}
    assert rejections(pools) == expected
