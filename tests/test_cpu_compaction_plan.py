"""The host half of b200vis_compact_topology, checked on CPU through the compaction step of b200vis_host_edit_plan.

A compaction keeps the live rows and the dead rows that held results still name, applies reparents that may break the
row order, renumbers the survivors in b200vis_plan_row_order's order and installs the plan set_topology would build.
So after any script the kept plan must equal the fresh plan (host_tile_plan / host_warp_plan) of the parent array a
plain model of the script produces, pass the checkers of a fresh plan, and keep planning edits correctly afterwards."""
import numpy as np

import bevy_b200 as bb
from bevy_b200 import abi, scenes

from test_cpu_incremental_plan import (DETACHED, HIERARCHY_CYCLE, INVALID_ARG, NO_PARENT, OK, World, check_edited,
                                       random_forest, random_step)

NONE = 0xFFFFFFFF
# check_edited patches abi.host_tile_plan / host_warp_plan for the rest of a test: the fresh planners, bound here
fresh_tile_plan, fresh_warp_plan = abi.host_tile_plan, abi.host_warp_plan


def compact(w, reparent=(), new_parent=(), held=()):
    """The model: (compacted World, old_to_new)."""
    n = w.n
    par = list(w.parent)
    for r, p in zip(reparent, new_parent):
        par[r] = int(p)
    held = set(int(h) for h in held)
    surv = [r for r in range(n) if w.alive[r] or r in held]
    s_of = {r: i for i, r in enumerate(surv)}
    ps = np.asarray([s_of[par[r]] if par[r] < n else par[r] for r in surv], np.uint32)
    new_to_old = [surv[i] for i in bb.plan_row_order(ps).tolist()]
    o2n = np.full(n, NONE, np.int64)
    o2n[new_to_old] = np.arange(len(new_to_old))
    out = World([o2n[par[r]] if par[r] < n else par[r] for r in new_to_old])
    out.alive = [w.alive[r] for r in new_to_old]
    return out, o2n


def descendants(w, r):
    kids = w.children()
    out, stack = set(), [r]
    while stack:
        x = stack.pop()
        out.add(x)
        stack += kids[x]
    return out


def copy_world(w):
    c = World(w.parent)
    c.alive = list(w.alive)
    return c


def random_compaction(rng, w, n_reparent=4, held_fraction=0.3):
    """Reparents onto any live row that is not in the row's own subtree (later rows preferred), and a random part of the
    dead rows held."""
    w = copy_world(w)
    live = [r for r in range(w.n) if w.alive[r]]
    reparent, new_parent = [], []
    for r in rng.choice(live, size=min(n_reparent, len(live)), replace=False).tolist() if live else []:
        k = rng.random()
        if k < 0.15:
            p = NO_PARENT
        elif k < 0.25:
            p = DETACHED
        else:
            sub = descendants(w, r)
            cands = [x for x in live if x not in sub and x > r] or [x for x in live if x not in sub]
            p = int(rng.choice(cands)) if cands else NO_PARENT
        reparent.append(int(r)); new_parent.append(p)
        w.parent[r] = p          # later picks see this reparent: no cycle through two of them
    dead = [r for r in range(w.n) if not w.alive[r]]
    held = [int(d) for d in dead if rng.random() < held_fraction]
    return reparent, new_parent, held


def run_mixed(parent, rng, n_rounds, monkeypatch, tile_rows, edits_per_round=3, **kw):
    """Rounds of random edit steps, each followed by a compaction; the plan is checked after every compaction and after
    the last edit."""
    w = World(parent)
    steps = []
    for _ in range(n_rounds):
        for _ in range(edits_per_round):
            s = random_step(rng, w, **kw)
            steps.append(s)
            w.apply(*s)
        reparent, new_parent, held = random_compaction(rng, w)
        steps.append(abi.Compaction(reparent, new_parent, held))
        w, _ = compact(w, reparent, new_parent, held)
        check_compacted(abi.host_edit_plan(parent, steps, max_rows=10 ** 7, tile_rows=tile_rows), w, monkeypatch, tile_rows)
    # an edit after the compactions: spawns and despawns (an order-keeping reparent may meet the 128 parent slots of a
    # full tile, which the edit refuses)
    s = random_step(rng, w, **dict(kw, n_reparent=0))
    steps.append(s)
    w.apply(*s)
    plan = abi.host_edit_plan(parent, steps, max_rows=10 ** 7, tile_rows=tile_rows)
    assert plan.rc == OK and plan.counters[3] == len(steps)
    check_edited(plan, w, monkeypatch, tile_rows)
    return w


def check_compacted(plan, w, monkeypatch, tile_rows):
    """The kept plan after a compaction is the fresh plan of the compacted parent array."""
    parent = np.asarray(w.parent, np.uint32)
    assert plan.rc == OK and plan.n == w.n
    desc8, topo = plan.tile_desc()
    f_desc, f_topo = fresh_tile_plan(parent, tile_rows)
    assert np.array_equal(desc8, f_desc) and np.array_equal(topo, f_topo)
    wd, nonroot, sched, wtopo = plan.warp_plan()
    fw = fresh_warp_plan(parent, tile_rows)
    for a, b in zip((wd, nonroot, sched, wtopo), fw):
        assert np.array_equal(a, b)
    check_edited(plan, w, monkeypatch, tile_rows)


def test_random_edits_and_compactions_equal_a_fresh_plan(monkeypatch):
    for seed in range(4):
        rng = np.random.default_rng(900 + seed)
        parent = random_forest(rng, int(rng.integers(300, 2000)))
        run_mixed(parent, rng, 2, monkeypatch, tile_rows=256)
        run_mixed(parent, rng, 2, monkeypatch, tile_rows=64)


def test_bench_forest_and_config1_trees(monkeypatch):
    rng = np.random.default_rng(11)
    for parent in (scenes.forest(n_trees=40, levels=8, n_lights=16).parent, scenes.propagate_bench_scene().parent):
        run_mixed(parent, rng, 1, monkeypatch, tile_rows=256, edits_per_round=2, n_despawn=4, n_reparent=2, n_spawn=30)


def test_the_order_is_plan_row_order_over_the_survivors():
    # a chain 0 <- 1 <- 2 and flat rows; row 1 dies with its child 2, row 4 moves under the later row 6 and row 5 is held:
    # survivors 0, 3, 4, 5, 6, 7 in current order, BFS -> 0, 3, 5 (held, detached), 6, 4 (child of 6), 7
    parent = np.asarray([NO_PARENT, 0, 1, NO_PARENT, NO_PARENT, NO_PARENT, NO_PARENT, NO_PARENT], np.uint32)
    steps = [([1, 2, 5], [], [], []), abi.Compaction([4], [6], [5])]
    plan = abi.host_edit_plan(parent, steps)
    assert plan.rc == OK and plan.n == 6
    want = np.asarray([NO_PARENT, NO_PARENT, DETACHED, NO_PARENT, 3, NO_PARENT], np.uint32)
    w = World(parent)
    w.apply(*steps[0])
    got, o2n = compact(w, [4], [6], [5])
    assert np.array_equal(np.asarray(got.parent, np.uint32), want)
    assert o2n.tolist() == [0, NONE, NONE, 1, 4, 2, 3, 5]
    assert np.array_equal(plan.tile_desc()[1], fresh_tile_plan(want)[1])


def test_reparents_onto_later_rows_give_a_topological_order(monkeypatch):
    rng = np.random.default_rng(4)
    parent = random_forest(rng, 1200)
    w = World(parent)
    live = list(range(w.n))
    # whole subtrees moved under rows after them, one of them under the last row
    moves = []
    for r in (3, 40, 500):
        sub = descendants(w, r)
        p = max(x for x in live if x not in sub)
        moves.append((r, p))
        w.parent[r] = p
    w = World(parent)
    reparent, new_parent = zip(*moves)
    plan = abi.host_edit_plan(parent, [abi.Compaction(reparent, new_parent)], tile_rows=256)
    got, o2n = compact(w, reparent, new_parent)
    p = np.asarray(got.parent, np.int64)
    real = p < len(p)
    assert (p[real] < np.nonzero(real)[0]).all()
    for r, q in moves:
        assert got.parent[o2n[r]] == o2n[q]
    check_compacted(plan, got, monkeypatch, 256)


def test_held_dead_rows_survive_and_the_others_are_dropped():
    rng = np.random.default_rng(8)
    parent = random_forest(rng, 700)
    w = World(parent)
    steps = []
    for _ in range(3):
        s = random_step(rng, w, n_despawn=6)
        steps.append(s)
        w.apply(*s)
    dead = [r for r in range(w.n) if not w.alive[r]]
    held = dead[::3]
    plan = abi.host_edit_plan(parent, steps + [abi.Compaction(held=held)])
    live = sum(w.alive)
    assert plan.rc == OK and plan.n == live + len(held)
    got, o2n = compact(w, held=held)
    assert all(o2n[d] != NONE for d in held) and all(o2n[d] == NONE for d in dead if d not in held)
    assert sum(not a for a in got.alive) == len(held)
    assert all(got.parent[o2n[d]] == DETACHED for d in held)
    # a second compaction with nothing held drops them
    plan2 = abi.host_edit_plan(parent, steps + [abi.Compaction(held=held), abi.Compaction()])
    assert plan2.rc == OK and plan2.n == live


def test_errors_leave_the_plan_unchanged():
    rng = np.random.default_rng(5)
    parent = random_forest(rng, 900)
    w = World(parent)
    good = []
    for _ in range(2):
        s = random_step(rng, w)
        good.append(s)
        w.apply(*s)
    ref = abi.host_edit_plan(parent, good)
    assert ref.rc == OK
    n = w.n
    kids = w.children()
    live = [r for r in range(n) if w.alive[r]]
    dead = [r for r in range(n) if not w.alive[r]]
    parent_row = next(r for r in live if kids[r])
    child = kids[parent_row][0]
    bad = {
        "cycle through a parent and its child": (abi.Compaction([parent_row], [child]), HIERARCHY_CYCLE),
        "reparent onto itself": (abi.Compaction([child], [child]), HIERARCHY_CYCLE),
        "two reparents that close a cycle": (abi.Compaction([live[0], live[1]], [live[1], live[0]]), HIERARCHY_CYCLE),
        "reparent a dead row": (abi.Compaction([dead[0]], [NO_PARENT]), INVALID_ARG),
        "reparent a row out of range": (abi.Compaction([n], [NO_PARENT]), INVALID_ARG),
        "new parent dead": (abi.Compaction([child], [dead[0]]), INVALID_ARG),
        "new parent out of range": (abi.Compaction([child], [n + 3]), INVALID_ARG),
        "reparent twice": (abi.Compaction([child, child], [NO_PARENT, DETACHED]), INVALID_ARG),
        "a live row held": (abi.Compaction(held=[live[0]]), INVALID_ARG),
        "a held row out of range": (abi.Compaction(held=[n]), INVALID_ARG),
    }
    for name, (step, code) in bad.items():
        got = abi.host_edit_plan(parent, good + [step])
        assert got.rc == code, name
        assert got.counters[3] == len(good) and got.n == ref.n, name
        for a, b in ((got.desc, ref.desc), (got.sched, ref.sched), (got.topo, ref.topo), (got.wtopo, ref.wtopo)):
            assert np.array_equal(a, b), name


def test_a_forest_made_two_pass_by_one_spawned_child_returns_to_one_pass():
    parent = scenes.forest(n_trees=3922, levels=8, n_lights=256).parent      # the bench world, ~1 M rows
    n = len(parent)
    leaf = 254                                                              # a leaf of the first tree
    grown = abi.host_edit_plan(parent, [([], [], [], [leaf])])
    assert grown.rc == OK and grown.counters[2] == 2
    plan = abi.host_edit_plan(parent, [([], [], [], [leaf]), abi.Compaction()])
    assert plan.rc == OK and plan.n == n + 1 and plan.counters[2] == 1
    # the new child now sits right after its tree's other rows of its level, inside the tree's tile
    fresh = fresh_tile_plan(np.asarray(compact(World(list(parent) + [leaf]))[0].parent, np.uint32))[0]
    assert len(plan.desc) == len(fresh)
