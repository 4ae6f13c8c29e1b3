"""The shapes row_certificate_sets names, checked on the host with the row oracles (subgraph_oracle,
basket_oracle, price_arb_oracle), so that a change to a generator fails without a GPU."""
import numpy as np
import pytest

import basket_oracle as bo
import price_arb_oracle as pa
import row_certificate_sets as rc
import subgraph_oracle as so


@pytest.fixture(scope="module")
def wide():
    return rc.wide_set(None)


@pytest.fixture(scope="module")
def deep():
    return rc.deep_set(None)


def row(ws, i, j, B):
    return so.row_subgraph(ws.lists(), j, i, ws.mask(B))


def test_wide_set_layout(wide):
    assert wide.p is None
    assert all(wide.mm[t] > 0 and wide.mt[t] > 0 for t in (rc.P, rc.G, rc.U))   # main and appended pools
    assert wide.retired and all(any(act for _, _, act in lst) for lst in wide.lists().values())
    assert sum(wide.m.values()) > 2500


def test_n_loc_shapes(wide):
    sh = rc.shapes()
    for n in rc.N_LOC:
        i, j, B = sh[f"n_loc={n}"]
        T, pools = row(wide, i, j, B)
        assert len(T) == n and T[:2] == [i, j], n
    # 257 and 258 local tokens: more than the CTA's 256 threads
    assert len(row(wide, *sh["n_loc=258"])[0]) == rc.SG_THREADS + 2


def test_pool_count_shapes(wide):
    sh = rc.shapes()
    for c in rc.POOL_COUNTS:
        T, pools = row(wide, *sh[f"pools={c}"])
        assert len(pools) == c, (c, len(pools))
    assert {rc.p2(c) for c in rc.POOL_COUNTS} == {256, 512, 1024}
    T, pools = row(wide, *sh["p2>=2048"])
    assert rc.p2(len(pools)) >= 2048 and len(T) == 258


def test_degree_shapes(wide):
    i, j, B = rc.shapes()["p2>=2048"]
    T, pools = row(wide, i, j, B)
    deg = rc.local_degrees(wide, pools, T)
    assert deg[i] > 256
    assert sum(33 <= deg[t] <= 64 for t in T) >= 3
    # the light rows: i holds more than 256 at n_loc = 258, and every B token few
    T, pools = row(wide, *rc.shapes()["n_loc=258"])
    deg = rc.local_degrees(wide, pools, T)
    assert deg[1] > 256 and max(deg[t] for t in T[2:]) <= 4


def test_k16_basket_and_limit_rows(wide):
    i, j, B = rc.shapes()["n_loc=258"]
    basket = [j] + B[:15]
    T, pools, unreachable = bo.row_basket(wide.lists(), basket, [1.0] * 16, i, wide.mask(B[15:]))
    assert len(basket) == 16 and set(basket) <= set(T) and not unreachable
    assert T[:17] == [i] + basket and len(T) == 258


def test_price_row_with_258_priced_tokens(wide):
    sh = rc.shapes(price=True)
    for name, (i, j, B) in sh.items():             # the price shapes hold the same counts
        T, pools = pa.row_order(wide.lists(), wide.mask([i, j] + B), np.ones(len(B) + 2))
        ref = row(wide, *rc.shapes()[name])
        assert len(T) == len(ref[0]) and len(pools) == len(ref[1]) and max(B) < rc.WIDE_N, name
    i, j, B = sh["n_loc=258"]
    toks = sorted([i, j] + B)
    T, pools = pa.row_order(wide.lists(), wide.mask(toks), np.ones(len(toks)))
    assert len(T) == 258 == len(toks)
    assert len(pools) == len(row(wide, i, j, B)[1])


def test_deep_set(deep):
    assert all(deep.mm[t] > 0 and deep.mt[t] > 0 for t in (rc.P, rc.G, rc.U))
    lists = deep.lists()
    for (a, b), cnt in rc.DEEP.items():
        assert len(lists[(a, b)]) == cnt
    R = np.concatenate([deep.main[t][0].ravel() for t in (rc.P, rc.G)] + [deep.tail[t][0].ravel() for t in (rc.P, rc.G)])
    assert R.min() < 1e-2 and R.max() > 1e8                         # reserves over 1e-3 .. 1e9 of value
    assert {0.05, 0.95} <= set(np.round(deep.w.ravel(), 2))
    for name, (i, j, B) in rc.deep_rows().items():
        T, pools = so.row_subgraph(lists, j, i, deep.mask(B))
        assert len(T) == len(B) + 2 and len(pools) >= 60, name
    T, pools = so.row_subgraph(lists, 8, 1, deep.mask(rc.deep_rows()["deep 1<-8 B=all"][2]))
    assert len(T) == 8 and max(rc.local_degrees(deep, pools, T).values()) > 200   # {5, 6}'s 200 pools
