"""Host checks of the per-row mask calls (include/cfmm_b200.h, "per-row masks"): the Python packing of
one token list per row into allow_off / allow_token and its argument errors, each row's token set and
pool list through the oracles with its own list as the mask on a batch of mixed lists, and the execute
levels over each row's own tokens against a pairwise conflict check.  No GPU."""
import itertools

import numpy as np
import pytest

import limit_order_oracle as lo
import row_mask_oracle as rm
import subgraph_oracle as so
from test_basket_orders_host import _Stub, lists


def test_packing(cr):
    pack = cr.router.pack_row_lists
    off, tok = pack([[3, 1], [], np.array([6, 2, 5])], 6, [(1, 2), (3, 4), (5, 6)], [256] * 3, "q")
    assert off.tolist() == [0, 2, 2, 5] and tok.tolist() == [3, 1, 6, 2, 5]
    assert off.dtype == np.int64 and tok.dtype == np.int64
    off, tok = pack([], 6, [], [], "q")
    assert off.tolist() == [0] and len(tok) == 0
    # the row's own tokens do not count against its room
    pack([[1, 2, 3]], 6, [(1, 2)], [1], "q")
    with pytest.raises(ValueError, match="more than 1"):
        pack([[3, 4]], 6, [(1, 2)], [1], "q")


@pytest.mark.parametrize("allowed, match", [
    ([[1]], "one token list per row"),
    ([[1], [0]], "outside 1..6"),
    ([[1], [7]], "outside 1..6"),
    ([[1], [2, 3, 2]], "listed twice"),
    ([[1], [1.5]], "integers"),
])
def test_packing_errors(cr, allowed, match):
    with pytest.raises(ValueError, match=match):
        cr.router.pack_row_lists(allowed, 6, [(1, 2), (3, 4)], [256, 256], "q")


def test_lists_select_the_rows_calls_and_keep_the_mask_errors(cr):
    assert cr.router.is_row_lists([[1, 2], []]) and cr.router.is_row_lists([np.array([3])]) and \
        cr.router.is_row_lists([])
    assert not cr.router.is_row_lists(np.ones(6, bool)) and not cr.router.is_row_lists([True, False, True])
    f = cr.DevicePools._subgraph
    with pytest.raises(ValueError, match="listed twice"):
        f(_Stub(), False, [1], [2], [1.0], [[3, 3]], None, None)
    with pytest.raises(ValueError, match="one token list per row"):
        f(_Stub(), False, [1, 3], [2, 4], [1.0, 1.0], [[3]], None, None)
    with pytest.raises(ValueError, match="allowed"):
        f(_Stub(), False, [1], [2], [1.0], None, None, None)
    with pytest.raises(ValueError, match="6 entries"):
        f(_Stub(), False, [1], [2], [1.0], np.ones(5, bool), None, None)
    # a basket row's room: CFMM_SUBGRAPH_MAX_TOKENS + 1 tokens besides token_out, entries included
    own, room = cr.router._basket_room(np.array([1, 2]), np.array([0, 1, 3]), np.array([3, 4, 5]))
    assert own == [[1, 3], [2, 4, 5]] and room == [256, 255]
    with pytest.raises(ValueError, match="outside 1..6"):
        cr.DevicePools._basket(_Stub(), False, [1], [0, 1], [3], [1.0], [[9]], None, None)
    with pytest.raises(ValueError, match="listed twice"):
        cr.DevicePools._limit(_Stub(), False, [1], [0, 1], [3], [1.0], [0.5], [[2, 2]], None, None)


def test_row_token_sets_and_pools_follow_each_rows_own_list():
    """A batch of rows with mixed lists (empty, holding the row's own tokens, overlapping): each row's T
    and pool list are the one-mask oracle's with that row's list as the mask, they depend only on the
    list as a set with the row's own tokens removed, and T lies in the row's own token set."""
    L = lists()
    n = 8
    sub_rows = [(2, 1, []), (2, 1, [3, 4]), (2, 1, [4, 3, 2, 1]), (7, 1, [2]), (5, 6, [1, 2, 3, 4, 7, 8]),
                (3, 4, [5, 6])]
    seen = []
    for j, i, lst in sub_rows:
        T, pools = so.row_subgraph(L, j, i, rm.row_mask(lst, n))
        T2, pools2 = so.row_subgraph(L, j, i, rm.row_mask(sorted(set(lst) - {j, i}), n))
        assert (T, pools) == (T2, pools2)
        assert set(T) <= rm.own_subgraph(j, i, lst)
        seen.append(T)
    assert seen[0] == [1] and seen[1] == [1, 2, 3, 4] and seen[2] == seen[1]
    assert seen[3] == [1] and seen[5] == [4, 3]
    lim_rows = [(1, [2], [1.0], [0.0], []), (1, [2, 7], [1.0, 1.0], [0.5, 0.0], [3, 4]),
                (1, [2, 5], [1.0, 1.0], [0.0, 2.0], [4, 3, 1])]
    for i, basket, amts, lims, lst in lim_rows:
        got = lo.row_limit(L, basket, amts, lims, i, rm.row_mask(lst, n))
        assert got == lo.row_limit(L, basket, amts, lims, i, rm.row_mask(set(lst) - {i} - set(basket), n))
        assert set(got[0]) <= rm.own_basket(i, basket, lst)
    assert lo.row_limit(L, [2], [1.0], [0.0], 1, rm.row_mask([], n))[2]          # 2 cut off from 1
    T, _, unreach, dropped, _ = lo.row_limit(L, [2, 5], [1.0, 1.0], [0.0, 2.0], 1, rm.row_mask([4, 3, 1], n))
    assert T == [1, 2, 3, 4] and not unreach and dropped == [False, True]


def brute_levels_ok(own, lev):
    """Pairwise: rows of one level share no token, conflicting rows keep batch order, and each row sits
    just above its latest-levelled conflicting predecessor."""
    for r, s in itertools.combinations(range(len(own)), 2):
        if own[r] & own[s]:
            assert lev[r] < lev[s]
        elif lev[r] == lev[s]:
            assert not own[r] & own[s]
    for s in range(len(own)):
        assert lev[s] == 1 + max([lev[r] for r in range(s) if own[r] & own[s]], default=0)


def test_levels_over_each_rows_own_tokens():
    rng = np.random.default_rng(5)
    for _ in range(50):
        q, n = int(rng.integers(1, 30)), int(rng.integers(4, 40))
        own = []
        for _ in range(q):
            j, i = rng.choice(n, size=2, replace=False) + 1
            lst = rng.choice(n, size=int(rng.integers(0, 4)), replace=False) + 1
            own.append(rm.own_subgraph(j, i, lst))
        brute_levels_ok(own, rm.levels(own))
    # disjoint rows share one level; a common token puts rows one after another
    own = [rm.own_subgraph(2 * r + 1, 2 * r + 2, []) for r in range(5)]
    assert rm.levels(own) == [1] * 5 and rm.launches(rm.levels(own), [False] * 5) == 1
    assert rm.launches(rm.levels(own), [False, True, False, True, False]) == 2
    own = [rm.own_basket(1, [2], [9]), rm.own_basket(3, [4], [9]), rm.own_basket(5, [6], [])]
    assert rm.levels(own) == [1, 2, 1]
