"""Column-group units of pruning's level and final rounds (DESIGN.md 4.9), restated in numpy.

predict_units_kernel splits a tile's row-block groups into column groups of 32 columns when the round's tiles cannot
fill the grid with row-block groups alone.  predict16_phase_b<1684, true, 1> then gives warp (wn, wm) the n8 tile wn
of column group cg over row slab wm; the unsplit unit gives warp wn all four n8 tiles j of columns wn * 32 .. + 31.
Here:
  (a) thread by thread, every part entry (ib, wm, g, column) is written by exactly one thread of exactly one column
      group, from the same V rows (wm * 32 + i * 8 + g, i ascending) and the same column as in the unsplit unit, and the
      B fragments a warp reads lie in the 32 columns its column group loads;
  (b) every (tile, row-block group, column group) is claimed once in the kernel's decode, a tile's arrival count is
      groups * column groups, every (row block, column group) is covered once, and exactly one unit per tile, the
      first column group of the group the kernel's warp argmin picks (the fewest k-tiles, the lower group on ties),
      computes mu.
The bit-equality of the finisher's order itself is restated in tests/test_prune_refine_cpu.py and
tests/test_prune_levels_cpu.py; with (a) it carries over to the column groups.
"""
import pytest

from test_prune_refine_cpu import unit_cut

PBM = PBN = 128
NT = 512


def thread_entries(nj, cg):
    """(wm, g, column) -> (V rows, column) of every accumulator pair a thread folds into s(ib), and the B columns read"""
    out, bcols = {}, set()
    for tid in range(NT):
        warp, lane = tid >> 5, tid & 31
        wn = warp >> 2
        wm = (warp + wn) & 3
        g, t4 = lane >> 2, lane & 3
        wc = wn * 32 if nj == 4 else cg * 32 + wn * 8
        for j in range(nj):
            bcols.add(wc + j * 8 + g)  # b[j]: B fragment column of lane (g, t4)
            for e in range(2):
                # m16n8k4: c0/c1 (c2/c3) of lane (g, t4) are column 2 t4 + e of the n8 tile, i.e. the B column that
                # lanes with g' = 2 t4 + e load as their b[j]
                col = wc + j * 8 + (2 * t4 + e)
                key = (wm, g, col)
                assert key not in out
                out[key] = (tuple(wm * 32 + i * 8 + g for i in range(4)), col)
    return out, bcols


def test_column_groups_cover_the_unsplit_entries():
    whole, _ = thread_entries(4, 0)
    assert len(whole) == 4 * 8 * PBN
    union = {}
    for cg in range(4):
        ent, bcols = thread_entries(1, cg)
        assert bcols == set(range(cg * 32, cg * 32 + 32))  # the loader's columns cb .. cb + 31 (cb = cg * 32)
        assert all(cg * 32 <= c < cg * 32 + 32 for (_, _, c) in ent)
        for k, v in ent.items():
            assert k not in union
            union[k] = v
    assert union == whole


def unit_cost(b0, nb, groups, j):
    a, b = unit_cut_from(b0, nb, groups, j), unit_cut_from(b0, nb, groups, j + 1)
    return (b * (b + 1) - a * (a + 1)) // 2


def unit_cut_from(b0, nb, groups, j):
    """unit_cut of predict16.cuh with a start block"""
    if j >= groups:
        return nb
    base, total = b0 * (b0 + 1) // 2, nb * (nb + 1) // 2 - b0 * (b0 + 1) // 2
    ib = b0
    while ib < nb and (ib * (ib + 1) // 2 - base) * groups < total * j:
        ib += 1
    return ib


def round_units(nt, b0, b1, colgroups, grid):
    """predict_units_kernel's groups and column groups of a level or final round (up to one row block per group)"""
    gmax = min(32, b1 - b0)
    cgs = colgroups if nt * gmax < 2 * grid else 1
    groups = max(1, min(gmax, 2 * grid // (nt * cgs)))
    return groups, cgs


def mu_group_shuffle(cost, groups):
    """the kernel's warp argmin: lanes >= groups hold INT64_MAX, xor butterfly 16 .. 1, the lower group on ties"""
    c = [cost[t] if t < groups else 2**63 - 1 for t in range(32)]
    j = list(range(32))
    for o in (16, 8, 4, 2, 1):
        oc = [c[t ^ o] for t in range(32)]
        oj = [j[t ^ o] for t in range(32)]
        for t in range(32):
            if oc[t] < c[t] or (oc[t] == c[t] and oj[t] < j[t]):
                c[t], j[t] = oc[t], oj[t]
    assert len(set(j)) == 1  # every lane agrees
    return j[0]


@pytest.mark.parametrize("nt,b0,b1,mu_expect", [
    (2, 8, 32, None),  # C3's final round
    (13, 4, 8, None),  # C3's level (keys from the stored interval: no mu unit)
    (1, 2, 8, 5),  # nb = 8, final: six groups of one row block, the last one empty
    (8, 8, 32, None), (128, 4, 8, None), (40, 1, 2, None),
])
def test_claims_arrivals_and_mu_unit(nt, b0, b1, mu_expect):
    grid = 132
    groups, cgs = round_units(nt, b0, b1, 4, grid)
    assert 1 <= groups <= 32 and cgs in (1, 4)
    cuts = [unit_cut_from(b0, b1, groups, j) for j in range(groups + 1)]
    assert cuts[0] == b0 and cuts[-1] == b1 and all(a <= b for a, b in zip(cuts, cuts[1:]))
    cost = [unit_cost(b0, b1, groups, j) for j in range(groups)]
    assert sum(cost) == (b1 * (b1 + 1) - b0 * (b0 + 1)) // 2
    mu_grp = mu_group_shuffle(cost, groups)
    if mu_expect is not None:
        assert mu_grp == mu_expect, (cuts, cost)
    seen, arrive, mu_units, blocks = set(), {}, {}, {}
    for u in range(nt * groups * cgs):  # the kernel's decode: row-block groups descending, tiles innermost
        tile, r = u % nt, u // nt
        grp, cg = groups - 1 - r // cgs, r % cgs
        assert (tile, grp, cg) not in seen
        seen.add((tile, grp, cg))
        arrive[tile] = arrive.get(tile, 0) + 1
        if grp == mu_grp and cg == 0:
            mu_units[tile] = mu_units.get(tile, 0) + 1
        for ib in range(cuts[grp], cuts[grp + 1]):
            blocks.setdefault(tile, []).append((ib, cg))
    assert all(a == groups * cgs for a in arrive.values()) and len(arrive) == nt
    assert all(m == 1 for m in mu_units.values()) and len(mu_units) == nt
    # every (row block, column group) of every tile is covered once: the part image is complete
    assert all(sorted(v) == [(ib, cg) for ib in range(b0, b1) for cg in range(cgs)] for v in blocks.values())
    if b1 - b0 <= 32 and nt * min(32, b1 - b0) * cgs <= 2 * grid:
        assert groups == b1 - b0  # room for one row block per group


@pytest.mark.parametrize("b0,b1,groups,expect", [
    (0, 32, 16, 6),  # C3's lead: no empty group, the lightest is the middle group [20, 21) of 21 k-tiles
    (2, 8, 4, 1),  # nb = 8 cut into four: [5, 6) of 6 k-tiles is the lightest
    (8, 32, 16, 15),  # an empty last group wins
])
def test_mu_group_of_non_split_cuts(b0, b1, groups, expect):
    cost = [unit_cost(b0, b1, groups, j) for j in range(groups)]
    assert mu_group_shuffle(cost, groups) == expect, cost
