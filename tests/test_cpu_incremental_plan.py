"""The incremental planner of b200vis_edit_topology, checked on CPU through b200vis_host_edit_plan.

After every edit step the kept plan must pass the invariants a fresh plan passes (the named-barrier replay and level
counts of test_cpu_tile_plan, the warp schedule, slot and pass checks of test_cpu_warp_plan), its topo words must decode
to the edited parent array (dead rows detached, T_HAS_CHILDREN = "has a live child"), an edit must re-plan only the
tiles it touches, and a failing edit must leave the plan exactly as it was."""
import numpy as np
import pytest

import bevy_b200 as bb
from bevy_b200 import abi, scenes

import test_cpu_tile_plan as tile_plan_tests
import test_cpu_warp_plan as warp_plan_tests

NO_PARENT, DETACHED = 0xFFFFFFFF, 0xFFFFFFFE
T_ROOT, T_HAS_CHILDREN, T_EXT_PARENT, T_DETACHED = 1 << 28, 1 << 29, 1 << 30, 1 << 31
OK, INVALID_ARG, HIERARCHY_CYCLE, CAPACITY, UNSUPPORTED = 0, 1, 4, 6, 8


class World:
    """The hierarchy an edit script produces: dead rows DETACHED, spawned rows appended."""

    def __init__(self, parent):
        self.parent = [int(p) for p in parent]
        self.alive = [True] * len(self.parent)

    @property
    def n(self):
        return len(self.parent)

    def children(self):
        kids = [[] for _ in range(self.n)]
        for r, p in enumerate(self.parent):
            if p < self.n:
                kids[p].append(r)
        return kids

    def apply(self, despawn, reparent, new_parent, spawn_parent):
        for d in despawn:
            self.parent[d] = DETACHED
            self.alive[d] = False
        for r, p in zip(reparent, new_parent):
            self.parent[r] = int(p)
        for p in spawn_parent:
            self.parent.append(int(p))
            self.alive.append(True)


def random_step(rng, w, n_despawn=3, n_reparent=3, n_spawn=5):
    """Recursive despawns, order-keeping reparents, spawns of roots, flat rows, children of old rows and of this batch."""
    live = [r for r in range(w.n) if w.alive[r]]
    kids = w.children()
    despawn = set()
    for r in rng.choice(live, size=min(n_despawn, len(live)), replace=False) if live else []:
        stack = [int(r)]
        while stack:
            x = stack.pop()
            if x not in despawn:
                despawn.add(x)
                stack += kids[x]
    despawn = sorted(despawn)
    dead = set(despawn)
    survivors = [r for r in live if r not in dead]
    reparent, new_parent = [], []
    for r in rng.choice(survivors, size=min(n_reparent, len(survivors)), replace=False) if survivors else []:
        r = int(r)
        k = rng.random()
        cands = [x for x in survivors[:survivors.index(r)] if r - x < 600]
        if k < 0.2 or not cands:
            p = NO_PARENT
        elif k < 0.3:
            p = DETACHED
        else:
            p = int(rng.choice(cands))
        reparent.append(r); new_parent.append(p)
    spawn_parent = []
    for j in range(n_spawn):
        k = rng.random()
        if k < 0.3 or not survivors:
            spawn_parent.append(NO_PARENT)
        elif k < 0.6:
            spawn_parent.append(int(rng.choice(survivors[-300:])))
        elif k < 0.7:
            spawn_parent.append(int(rng.choice(survivors)))
        elif j:
            spawn_parent.append(w.n + int(rng.integers(0, j)))
        else:
            spawn_parent.append(DETACHED)
    return despawn, reparent, new_parent, spawn_parent


def check_edited(plan, w, monkeypatch, tile_rows=0):
    parent = np.asarray(w.parent, np.uint32)
    n = len(parent)
    assert plan.rc == OK and plan.n == n
    topo = plan.topo
    # the topo words decode to the edited parent array
    desc8, _ = plan.tile_desc()
    base_of = np.zeros(n, np.int64)
    for base, nr, *_ in desc8.tolist():
        base_of[base:base + nr] = base
    has_live_child = np.zeros(n, bool)
    for r in range(n):
        p, t = int(parent[r]), int(topo[r])
        if p == NO_PARENT:
            assert t & T_ROOT
        elif p == DETACHED:
            assert t & T_DETACHED
        else:
            has_live_child[p] = True
            assert (t & T_EXT_PARENT) or base_of[r] + (t & 0x1FF) == p, f"row {r}: topo names the wrong parent"
            assert not (t & T_EXT_PARENT) or p < base_of[r]
    assert (((topo & T_HAS_CHILDREN) != 0) == has_live_child).all()
    for r in range(n):
        if not w.alive[r]:
            assert parent[r] == DETACHED and not has_live_child[r]
    # the invariants of a fresh plan, checked on the edited one by the fresh plan's own checkers
    monkeypatch.setattr(abi, "host_tile_plan", lambda p, tr=0: plan.tile_desc())
    tile_plan_tests.check(parent, tile_rows)
    monkeypatch.setattr(abi, "host_warp_plan", lambda p, tr=0: plan.warp_plan())
    warp_plan_tests.check_plan(parent, tile_rows)


def run_script(w0_parent, steps, monkeypatch, tile_rows=0, check_every=True):
    w = World(w0_parent)
    for i in range(len(steps)):
        w.apply(*steps[i])
        if check_every or i == len(steps) - 1:
            plan = abi.host_edit_plan(w0_parent, steps[:i + 1], tile_rows=tile_rows)
            assert plan.counters[3] == i + 1
            check_edited(plan, w, monkeypatch, tile_rows)
    return w


def random_forest(rng, n):
    parent = np.full(n, NO_PARENT, np.uint32)
    for r in range(1, n):
        k = rng.random()
        if k < 0.15:
            continue
        if k < 0.18:
            parent[r] = DETACHED
            continue
        parent[r] = rng.integers(max(0, r - int(rng.integers(1, 400))), r)
    order = bb.plan_row_order(parent)
    inv = np.empty(n, np.int64); inv[order] = np.arange(n)
    p2 = parent[order].astype(np.int64)
    real = p2 < n
    p2[real] = inv[p2[real]]
    return p2.astype(np.uint32)


def random_steps(rng, parent, k, **kw):
    w = World(parent)
    steps = []
    for _ in range(k):
        s = random_step(rng, w, **kw)
        steps.append(s)
        w.apply(*s)
    return steps


@pytest.mark.parametrize("seed", range(6))
def test_random_forests_random_edits(seed, monkeypatch):
    rng = np.random.default_rng(700 + seed)
    parent = random_forest(rng, int(rng.integers(200, 2500)))
    steps = random_steps(rng, parent, 6)
    run_script(parent, steps, monkeypatch)
    run_script(parent, steps, monkeypatch, tile_rows=64, check_every=False)


def test_bench_forest_and_config1_trees(monkeypatch):
    rng = np.random.default_rng(3)
    for parent in (scenes.forest(n_trees=40, levels=8, n_lights=16).parent, scenes.propagate_bench_scene().parent):
        steps = random_steps(rng, parent, 4, n_despawn=2, n_reparent=2, n_spawn=20)
        run_script(parent, steps, monkeypatch, check_every=False)


def test_deep_chain(monkeypatch):
    chain = np.concatenate([[NO_PARENT], np.arange(699)]).astype(np.uint32)
    steps = [
        ([699], [], [], [698, 700, 701]),             # cut the leaf, grow the chain by three
        ([], [300], [NO_PARENT], [299]),              # split it in two, hang a leaf off the upper part
        ([700, 701, 702], [], [], [NO_PARENT] * 3),   # drop the grown tail (recursive), three flat rows
    ]
    run_script(chain, steps, monkeypatch)


def test_spawn_children_of_the_same_batch_and_flat_rows(monkeypatch):
    parent = np.full(300, NO_PARENT, np.uint32)
    steps = [([], [], [], [NO_PARENT, 300, 301, 301, 5, DETACHED]),
             ([301], [302, 303], [300, NO_PARENT], []),    # 301 has children 302, 303: they are reparented -- too late
             ]
    plan = abi.host_edit_plan(parent, steps)
    assert plan.rc == INVALID_ARG and plan.counters[3] == 1
    steps[1] = ([303], [302], [300], [])
    run_script(parent, steps, monkeypatch)


def test_one_spawned_leaf_replans_at_most_two_tiles():
    parent = scenes.forest(n_trees=3922, levels=8, n_lights=256).parent      # the bench world, ~1 M rows
    n = len(parent)
    leaf = 254                                                              # last row of the first tree: a leaf
    assert (parent != leaf).all()
    plan = abi.host_edit_plan(parent, [([], [], [], [leaf])])
    tiles, rows, passes, steps = plan.counters
    assert plan.rc == OK and steps == 1 and plan.n == n + 1
    assert tiles <= 2 and rows <= 512, plan.counters
    assert passes == 2                                                      # the new child's tile runs after its parent's
    plan = abi.host_edit_plan(parent, [([], [], [], [NO_PARENT])])
    assert plan.counters[0] <= 1 and plan.counters[1] <= 256 and plan.counters[2] == 1


def test_errors_leave_the_plan_unchanged():
    rng = np.random.default_rng(5)
    parent = random_forest(rng, 900)
    good = random_steps(rng, parent, 2)
    ref = abi.host_edit_plan(parent, good)
    assert ref.rc == OK
    w = World(parent)
    for s in good:
        w.apply(*s)
    n = w.n
    kids = w.children()
    live = [r for r in range(n) if w.alive[r]]
    dead = [r for r in range(n) if not w.alive[r]]
    with_kids = next(r for r in live if kids[r])
    leaf = next(r for r in live if not kids[r] and r > 10)
    bad = {
        "capacity": (([], [], [], [NO_PARENT] * 3), CAPACITY, n + 2),
        "despawn out of range": (([n], [], [], []), INVALID_ARG, None),
        "despawn dead row": (([dead[0]], [], [], []), INVALID_ARG, None),
        "despawn twice": (([leaf, leaf], [], [], []), INVALID_ARG, None),
        "despawn with live children": (([with_kids], [], [], []), INVALID_ARG, None),
        "reparent dead row": (([], [dead[0]], [NO_PARENT], []), INVALID_ARG, None),
        "reparent despawned row": (([leaf], [leaf], [NO_PARENT], []), INVALID_ARG, None),
        "reparent onto a later row": (([], [leaf], [leaf + 1 if leaf + 1 < n else leaf], []), UNSUPPORTED, None),
        "reparent onto itself": (([], [leaf], [leaf], []), UNSUPPORTED, None),
        "reparent onto a dead row": (([], [n - 1 if w.alive[n - 1] else live[-1]], [dead[0]], []), INVALID_ARG, None),
        "reparent twice": (([], [leaf, leaf], [NO_PARENT, DETACHED], []), INVALID_ARG, None),
        "spawn under a dead row": (([], [], [], [dead[0]]), INVALID_ARG, None),
        "spawn under a later row of the batch": (([], [], [], [n + 1, NO_PARENT]), UNSUPPORTED, None),
        "spawn parent out of range": (([], [], [], [n + 7]), INVALID_ARG, None),
    }
    for name, (step, code, max_rows) in bad.items():
        got = abi.host_edit_plan(parent, good + [step], max_rows=max_rows if max_rows else n + 10)
        assert got.rc == code, name
        assert got.counters[3] == len(good) and got.n == ref.n, name
        for a, b in ((got.desc, ref.desc), (got.sched, ref.sched), (got.topo, ref.topo), (got.wtopo, ref.wtopo)):
            assert np.array_equal(a, b), name


def test_reparent_that_overflows_the_warp_parent_slots_is_unsupported():
    # one 256-row tile: a 128-row chain (127 rows with in-tile children) and 128 flat rows; two new parents among the flat
    # rows would need 129 of the warp kernel's 128 parent slots
    parent = np.full(256, NO_PARENT, np.uint32)
    parent[1:128] = np.arange(0, 127)
    plan = abi.host_edit_plan(parent, [])
    assert len(plan.desc) == 1 and ((plan.wtopo >> 22) & 1).sum() == 127
    assert abi.host_edit_plan(parent, [([], [200], [150], [])]).rc == OK
    got = abi.host_edit_plan(parent, [([], [200, 201], [150, 151], [])])
    assert got.rc == UNSUPPORTED and np.array_equal(got.topo, plan.topo) and np.array_equal(got.desc, plan.desc)
