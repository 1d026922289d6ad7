"""Oracle restatements of the SURVEY.md 8(f) rows, pinned on the reference's own tests where it has any and
cross-checked against independent numpy restatements elsewhere (CPU only)."""
import numpy as np
import pytest

from oracle import oracle as orc

INH, HID, VIS, NOC = orc.VIS_INHERITED, orc.VIS_HIDDEN, orc.VIS_VISIBLE, orc.VIS_NO_COMPONENTS
NP = 0xFFFFFFFF


# ---- N1 ---------------------------------------------------------------------------------------------
def test_n1_pair_lookup_uses_main_entity_sort_order():
    """crates/bevy_render/src/view/visibility/mod.rs:436-481"""
    main_a, main_b = 1, 2
    render_a, render_b = 2, 1   # render entities sort differently from the main entities
    render, main = orc.sort_pairs_by_main([render_a, render_b], [main_a, main_b])
    a_r, a_m, r_r, r_m = orc.update_cpu_culled_entities([], [], render, main)
    pairs_full_sort = sorted([(render_a, main_a), (render_b, main_b)])
    got = list(zip(render.tolist(), main.tolist()))
    assert got != pairs_full_sort
    assert got == sorted([(render_a, main_a), (render_b, main_b)], key=lambda p: p[1])
    assert list(zip(a_r.tolist(), a_m.tolist())) == got and len(r_m) == 0
    for e, m in got:
        assert orc.entity_pair_is_visible(render, main, e, m)
    assert not orc.entity_pair_is_visible(render, main, render_a, main_b)


@pytest.mark.parametrize("seed", range(5))
def test_n1_diff_matches_set_algebra(seed):
    rng = np.random.default_rng(seed)
    universe = rng.choice(1 << 40, size=3000, replace=False).astype(np.uint64)
    old = np.sort(universe[rng.random(3000) < 0.5])
    new = np.sort(universe[rng.random(3000) < 0.5])
    if seed == 0:
        old = old[:0]
    if seed == 1:
        new = new[:0]
    a_r, a_m, r_r, r_m = orc.update_cpu_culled_entities(old + 7, old, new + 7, new)
    assert np.array_equal(a_m, np.setdiff1d(new, old)) and np.array_equal(a_r, a_m + 7)
    assert np.array_equal(r_m, np.setdiff1d(old, new)) and np.array_equal(r_r, r_m + 7)


# ---- N2 ---------------------------------------------------------------------------------------------
def _csr(rng, n_clusters, n_lights, mean):
    counts = rng.poisson(mean, n_clusters).astype(np.uint32)
    counts = np.minimum(counts, n_lights)
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.uint32)
    indices = np.concatenate([np.sort(rng.choice(n_lights, c, replace=False)) for c in counts] + [np.zeros(0, np.int64)])
    return offsets, indices.astype(np.uint32)


def test_n2_storage_layout():
    rng = np.random.default_rng(1)
    offsets, indices = _csr(rng, 3672, 256, 3.0)
    gmap = rng.permutation(256).astype(np.uint32)
    oc, il, no, ni = orc.cluster_bindings(offsets, indices, gmap, storage=True)
    assert no == 3672 and ni == offsets[-1]
    assert np.array_equal(oc[:, 0], offsets[:-1]) and np.array_equal(oc[:, 1], np.diff(offsets))
    assert not oc[:, 2:].any()
    assert np.array_equal(il, gmap[indices])


@pytest.mark.parametrize("mean", [1.0, 6.0])
def test_n2_uniform_layout_and_overflow(mean):
    rng = np.random.default_rng(2)
    offsets, indices = _csr(rng, 3672, 200, mean)
    total = int(offsets[-1])
    oc, il, no, ni = orc.cluster_bindings(offsets, indices, None, storage=False)
    counts = np.diff(offsets)
    if total <= 16384:
        assert mean == 1.0 and ni == total and no == 3672
        last = 3671
    else:
        assert ni == 16384
        last = int(np.searchsorted(offsets, 16384, side="right") - 1)   # the cluster that holds index slot 16384
        assert no == last + 1
    want = np.zeros(4096, np.uint32)
    c = np.arange(last + 1)
    want[c] = ((offsets[c] & 0x3FFF) << 18) | ((counts[c] & 0x1FF) << 9)
    assert np.array_equal(oc, want)
    packed = np.zeros(16384, np.uint8)
    packed[:ni] = indices[:ni]
    assert np.array_equal(il, packed.view("<u4"))


def view_cluster_bindings_literal(offsets, indices, entity_to_index, storage):
    """prepare_clusters_for_cpu_clustering (bevy_pbr/src/cluster/mod.rs:494-534) over the record stream of
    extract_clusters_for_cpu_clustering (:419-470), one record at a time into ViewClusterBindings (:596-705).
    `entity_to_index` maps a light ordinal to its GPU index; an ordinal missing from it takes the dummy path."""
    MAX_INDICES, MAX_UNIFORM_ITEMS = 16384, 16384 // 4 // 4
    records = []
    for c in range(len(offsets) - 1):
        records.append(("header", int(offsets[c + 1] - offsets[c])))
        records += [("light", int(e)) for e in indices[offsets[c]:offsets[c + 1]]]
    st = dict(n_offsets=0, n_indices=0)
    if storage:
        oc, il = [], []
    else:
        oc = [[0] * 4 for _ in range(MAX_UNIFORM_ITEMS)]        # clear()
        il = [[0] * 4 for _ in range(MAX_UNIFORM_ITEMS)]

    def push_offset_and_counts(offset, point_lights):
        if storage:
            oc.append([offset, point_lights, 0, 0, 0, 0, 0, 0])
        else:
            array_index = st["n_offsets"] >> 2
            if array_index < MAX_UNIFORM_ITEMS:
                oc[array_index][st["n_offsets"] & 3] = ((offset & 0x3FFF) << 18) | ((point_lights & 0x1FF) << 9) | (0 & 0x1FF)
        st["n_offsets"] += 1

    def push_raw_index(index):
        n = st["n_indices"]
        if storage:
            il.append(index)
        else:
            il[n >> 4][(n >> 2) & 3] |= (index << (8 * (n & 3))) & 0xFFFFFFFF   # u32 shift: the high bits fall off
        st["n_indices"] += 1

    for kind, value in records:
        if kind == "header":
            push_offset_and_counts(st["n_indices"], value)
            continue
        index = entity_to_index.get(value)
        if index is None:
            if not storage and st["n_indices"] >= MAX_INDICES:
                break                     # data[array_index] past the array: the reference panics here
            push_raw_index(0xFFFFFFFF)    # push_dummy_index
            continue
        if st["n_indices"] >= MAX_INDICES and not storage:
            break
        push_raw_index(index)
    if storage:
        return np.array(oc, np.uint32).reshape(-1, 8), np.array(il, np.uint32), st["n_offsets"], st["n_indices"]
    return np.array(oc, np.uint32).reshape(-1), np.array(il, np.uint32).reshape(-1), st["n_offsets"], st["n_indices"]


def binding_csr(case):
    """Hand-built CSRs (offsets, indices, cluster count) for the packing limits."""
    rng = np.random.default_rng(len(case))
    if case.startswith("total_"):                  # 16383 / 16384 / 16385 indices, the last cluster closing the stream
        total = int(case[6:])
        counts = np.full(total // 7, 7); counts = np.concatenate([counts, [total - counts.sum()]])
        counts = np.insert(counts, rng.integers(0, len(counts), 40), 0)
    elif case == "break_then_empty":               # the 16384th index closes a cluster; then empty clusters, then lights
        counts = np.concatenate([np.full(16384 // 8, 8), [0, 0, 0, 5, 0, 3]])
    elif case == "break_mid_cluster":              # index 16384 falls inside a cluster
        counts = np.concatenate([np.full(2047, 8), [12, 0, 4]])
    elif case == "counts_511_512_600":             # the 9-bit count field: 511 fits, 512 wraps to 0, 600 to 88
        counts = np.array([3, 511, 0, 512, 1, 600, 2])
    else:
        raise KeyError(case)
    counts = counts.astype(np.int64)
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.uint32)
    indices = rng.integers(0, 700, int(offsets[-1])).astype(np.uint32)   # ordinals up to 699: past 255 and past a short map
    return offsets, indices


BINDING_CASES = ["total_16383", "total_16384", "total_16385", "break_then_empty", "break_mid_cluster", "counts_511_512_600"]


@pytest.mark.parametrize("storage", [True, False])
@pytest.mark.parametrize("mapping", ["identity", "full", "short"])
@pytest.mark.parametrize("case", BINDING_CASES)
def test_n2_bindings_at_the_packing_limits_equal_the_record_loop(case, mapping, storage):
    offsets, indices = binding_csr(case)
    rng = np.random.default_rng(7)
    if mapping == "identity":
        gmap, e2i = None, {o: o for o in range(700)}
    else:
        n_map = 700 if mapping == "full" else 300
        gmap = rng.permutation(1000)[:n_map].astype(np.uint32)      # GPU indices up to 999: more than 8 bits
        e2i = {o: int(gmap[o]) for o in range(n_map)}
    got = orc.cluster_bindings(offsets, indices, gmap, storage=storage)
    want = view_cluster_bindings_literal(offsets, indices, e2i, storage)
    assert got[2:] == want[2:], f"n_offsets / n_indices {got[2:]} vs {want[2:]}"
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    total, counts = int(offsets[-1]), np.diff(offsets)
    # each case reaches the limit it is named for
    if not storage:
        assert want[3] == min(total, 16384)
        assert want[2] == np.count_nonzero(offsets[:-1] <= 16384)
    if case.startswith("total_"):
        assert total == int(case[6:])
    if case == "break_then_empty":
        assert (offsets[:-1] == 16384).sum() == 4 and counts[offsets[:-1] == 16384].tolist() == [0, 0, 0, 5]
    if case == "counts_511_512_600" and not storage:
        assert [(w >> 9) & 0x1FF for w in want[0][[1, 3, 5]]] == [511, 0, 88]
    if mapping != "identity" and storage:
        assert (want[1] > 255).any()
    if mapping == "short" and storage:
        assert (want[1] == 0xFFFFFFFF).any()


# ---- N4a --------------------------------------------------------------------------------------------
def test_n4_visibility_ranges_against_numpy():
    rng = np.random.default_rng(3)
    n = 4000
    gt = rng.normal(size=(n, 12)).astype(np.float32) * 20
    bounds = rng.normal(size=(n, 6)).astype(np.float32)
    flags = (rng.integers(0, 2, n) * orc.F_HAS_AABB | rng.integers(0, 2, n) * orc.F_HAS_VIS_RANGE
             | (rng.random(n) < 0.1) * orc.F_NO_CPU_CULLING).astype(np.uint8)
    start = rng.uniform(0, 40, n).astype(np.float32)
    rng_se = np.stack([start, start + rng.uniform(0, 60, n).astype(np.float32)], 1)
    use_aabb = rng.integers(0, 2, n).astype(np.uint8)
    views = rng.normal(size=(40, 3)).astype(np.float32) * 30   # > 32: only the first 32 count
    got = orc.check_visibility_ranges(gt, bounds, flags, rng_se, use_aabb, views)
    f32 = np.float32
    c = bounds[:, :3]
    tp = np.stack([((gt[:, k] * c[:, 0] + gt[:, 3 + k] * c[:, 1]) + gt[:, 6 + k] * c[:, 2]) + gt[:, 9 + k] for k in range(3)], 1)
    pos = np.where(((use_aabb != 0) & ((flags & orc.F_HAS_AABB) != 0))[:, None], tp, gt[:, 9:12]).astype(f32)
    want = np.zeros(n, np.uint32)
    for v in range(32):
        d = views[v][None, :] - pos
        dist = np.sqrt(((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]).astype(f32)).astype(f32)
        want |= ((dist >= rng_se[:, 0]) & (dist < rng_se[:, 1])).astype(np.uint32) << np.uint32(v)
    want[((flags & orc.F_HAS_VIS_RANGE) == 0) | ((flags & orc.F_NO_CPU_CULLING) != 0)] = 0
    assert np.array_equal(got, want)
    assert got.any() and (got == 0).any()


# ---- N4b --------------------------------------------------------------------------------------------
def _run(parent, vis, inh, changed_rows, removed=()):
    return orc.visibility_propagate(parent, vis, inh, changed_rows, removed)


def test_n4_visibility_propagation():
    """visibility/mod.rs:950-1040: two five-node trees"""
    #        root1 c1 c2 g1(c1) g2(c2) | root2 c1 c2 g1 g2
    parent = [NP, 0, 0, 1, 2, NP, 5, 5, 6, 7]
    vis = [HID, INH, HID, INH, INH, INH, INH, HID, INH, INH]
    inh, _ = _run(parent, vis, np.zeros(10, np.uint8), np.arange(10))
    assert inh.tolist() == [0, 0, 0, 0, 0, 1, 1, 0, 1, 0]


def test_n4_on_parent_change_and_removed():
    """visibility/mod.rs:1042-1090 and :1092-1128"""
    parent = [NP, NP, 0, 0]           # parent1 (Hidden), parent2 (Visible), child1, child2
    vis = [HID, VIS, INH, INH]
    inh, _ = _run(parent, vis, np.zeros(4, np.uint8), np.arange(4))
    parent[3] = 1                     # child2 re-parented to parent2; parent2's Visibility re-inserted
    inh, _ = _run(parent, vis, inh, [1, 3])
    assert inh[2] == 0 and inh[3] == 1
    parent = [NP, 0]
    vis = [HID, INH]
    inh, _ = _run(parent, vis, np.zeros(2, np.uint8), [0, 1])
    assert inh[1] == 0
    inh, _ = _run([NP, NP], vis, inh, [], removed=[1])
    assert inh[1] == 1


def test_n4_unconditional_visible_and_invalid_parent():
    """visibility/mod.rs:1130-1190 and :1268-1283"""
    parent = [NP, 0, 0, 1, 2, NP, NP]
    vis = [VIS, INH, HID, VIS, VIS, INH, HID]
    inh, _ = _run(parent, vis, np.zeros(7, np.uint8), np.arange(7))
    assert inh.tolist() == [1, 1, 0, 1, 1, 1, 0]
    inh, _ = _run([NP, 0], [NOC, INH], np.zeros(2, np.uint8), [1])
    assert inh[1] == 1


def test_n4_change_detection_sequence():
    """visibility/mod.rs:1192-1266: id1 -> id2 -> id3 (Hidden) -> id4"""
    parent = [NP, 0, 1, 2]
    vis = np.array([INH, INH, HID, INH], np.uint8)
    inh, _ = _run(parent, vis, np.zeros(4, np.uint8), np.arange(4))
    vis[0] = HID
    inh, ch = _run(parent, vis, inh, [0])
    assert ch.tolist() == [1, 1, 0, 0]
    inh, ch = _run(parent, vis, inh, [])
    assert not ch.any()
    vis[2] = INH
    inh, ch = _run(parent, vis, inh, [2])
    assert not ch.any()
    vis[1] = VIS
    inh, ch = _run(parent, vis, inh, [1])
    assert ch.tolist() == [0, 1, 1, 1]
    inh, ch = _run(parent, vis, inh, [])
    assert not ch.any()


def fixpoint(parent, vis):
    """What the device computes: the closed form the change-driven system converges to."""
    n = len(parent)
    out = np.zeros(n, np.uint8)
    for i in range(n):   # parents precede children in these tests
        if vis[i] & NOC:
            continue
        k = vis[i] & 3
        p = parent[i]
        out[i] = 1 if k == VIS else 0 if k == HID else (out[p] if p != NP and not (vis[p] & NOC) else 1)
    return out


@pytest.mark.parametrize("seed", range(4))
def test_n4_change_driven_equals_fixpoint_on_random_edits(seed):
    rng = np.random.default_rng(seed)
    n = 600
    parent = np.array([NP if i < 8 or rng.random() < 0.02 else rng.integers(0, i) for i in range(n)], np.uint32)
    vis = rng.choice([INH, INH, INH, HID, VIS], n).astype(np.uint8)
    inh, _ = _run(parent, vis, np.zeros(n, np.uint8), np.arange(n))
    assert np.array_equal(inh, fixpoint(parent, vis))
    for _ in range(12):
        rows = rng.choice(n, 10, replace=False)
        vis[rows] = rng.choice([INH, HID, VIS], 10)
        before = inh.copy()
        inh, ch = _run(parent, vis, inh, np.sort(rows))
        assert np.array_equal(inh, fixpoint(parent, vis))
        assert np.array_equal(ch != 0, inh != before)


# ---- N3 ---------------------------------------------------------------------------------------------
def test_n3_cubemap_frusta_host_equals_oracle_and_faces_look_along_their_axes():
    """update_point_light_frusta (bevy_light/src/point_light.rs:212-265): the product's host helper and the oracle are
    separate restatements and must agree bit for bit; each face sees a point 5 units along its own axis only."""
    from bevy_b200 import abi
    rng = np.random.default_rng(0)
    axes = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, -1], [0, 0, 1]], np.float32)   # CUBE_MAP_FACES
    for i in range(40):
        q = rng.normal(size=4); q /= np.linalg.norm(q)
        trs = np.concatenate([rng.uniform(-50, 50, 3), q, rng.uniform(0.5, 2, 3)]).astype(np.float32)
        gt = orc.affine_from_trs(trs)
        a = orc.point_light_frusta(gt, 17.5, 0.1)
        b = abi.host_point_light_frusta(gt, 17.5, 0.1)
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
        assert np.allclose(np.linalg.norm(a[..., :3], axis=-1), 1.0, atol=1e-6)
        for f in range(6):
            for k in range(6):
                p = gt[9:12] + 5 * axes[k]
                assert orc.intersects_sphere(a[f], p, 0.01, True) == (f == k)
            # the far plane is shared by the six faces: `range` behind the light along the light's own back direction
            assert np.array_equal(a[f, 5], a[0, 5])


def test_n3_point_light_mesh_visibility_against_a_plain_loop():
    rng = np.random.default_rng(11)
    n, L = 500, 5
    q = rng.normal(size=(n, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True)
    trs = np.concatenate([rng.uniform(-30, 30, (n, 3)), q, rng.uniform(0.5, 2, (n, 3))], 1).astype(np.float32)
    gt = np.stack([orc.affine_from_trs(t) for t in trs])
    bounds = np.concatenate([rng.normal(size=(n, 3)) * 0.3, rng.uniform(0.2, 2.0, (n, 3))], 1).astype(np.float32)
    flags = (orc.F_INHERITED_VISIBLE * (rng.random(n) < 0.9) | orc.F_HAS_AABB * (rng.random(n) < 0.85)
             | orc.F_NO_FRUSTUM_CULLING * (rng.random(n) < 0.05) | orc.F_HAS_VIS_RANGE * (rng.random(n) < 0.3)
             | orc.F_NO_CPU_CULLING * (rng.random(n) < 0.05)).astype(np.uint8)
    caster = (rng.random(n) < 0.8).astype(np.uint8)
    layers = rng.integers(1, 4, n).astype(np.uint64)
    range_mask = rng.integers(0, 4, n).astype(np.uint32)
    bits = rng.permutation(n).astype(np.uint64) + 100
    vv0 = rng.choice([0, 2], n).astype(np.uint8)             # after reset_view_visibility: only the "previous" bit
    lpos = rng.uniform(-20, 20, (L, 3)).astype(np.float32); lrange = rng.uniform(8, 30, L).astype(np.float32)
    llayers = rng.integers(1, 4, L).astype(np.uint64)
    ident = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1], np.float32)
    frusta = np.stack([orc.point_light_frusta(np.concatenate([ident, lpos[l]]), lrange[l], 0.1) for l in range(L)])
    vv, ch = vv0.copy(), np.zeros(n, np.uint8)
    got = orc.check_point_light_mesh_visibility(gt, bounds, flags, caster, bits, vv, ch, np.concatenate([lpos, lrange[:, None]], 1),
                                                frusta, layer_mask=layers, range_mask=range_mask, lod_origin_index=1,
                                                light_layers=llayers)
    want_vis = np.zeros(n, bool)
    total = 0
    for l in range(L):
        lists = [[] for _ in range(6)]
        for r in range(n):
            f = int(flags[r])
            if not caster[r] or f & orc.F_NO_CPU_CULLING or not f & orc.F_INHERITED_VISIBLE:
                continue
            if not int(llayers[l]) & int(layers[r]):
                continue
            if f & orc.F_HAS_VIS_RANGE and not (range_mask[r] >> 1) & 1:
                continue
            faces = range(6)
            if f & orc.F_HAS_AABB:
                no_fc = bool(f & orc.F_NO_FRUSTUM_CULLING)
                if not no_fc and not orc.sphere_intersects_obb(lpos[l], lrange[l], bounds[r, :3], bounds[r, 3:], gt[r]):
                    continue
                faces = [k for k in range(6) if no_fc or orc.intersects_obb(frusta[l, k], bounds[r, :3], bounds[r, 3:], gt[r], True, True)]
            for k in faces:
                lists[k].append(r); want_vis[r] = True
        for k in range(6):
            want = np.array(sorted(lists[k], key=lambda r: bits[r]), np.uint32)
            assert np.array_equal(got[l][k], want)
            total += len(want)
    assert total > 50
    assert np.array_equal((vv & 1) != 0, want_vis)
    assert np.array_equal(ch != 0, want_vis & (vv0 == 0))    # change fires on hidden -> visible only
    orc.mark_newly_hidden(flags, vv, ch)
    gone = ((vv0 == 2) & ~want_vis & ((flags & orc.F_NO_CPU_CULLING) == 0))
    assert np.array_equal(vv[gone], np.zeros(gone.sum(), np.uint8)) and ch[gone].all()


def _shadow_world(seed, n=400):
    rng = np.random.default_rng(seed)
    q = rng.normal(size=(n, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True)
    trs = np.concatenate([rng.uniform(-30, 30, (n, 3)), q, rng.uniform(0.5, 2, (n, 3))], 1).astype(np.float32)
    gt = np.stack([orc.affine_from_trs(t) for t in trs])
    bounds = np.concatenate([rng.normal(size=(n, 3)) * 0.3, rng.uniform(0.2, 2.0, (n, 3))], 1).astype(np.float32)
    flags = (orc.F_INHERITED_VISIBLE * (rng.random(n) < 0.9) | orc.F_HAS_AABB * (rng.random(n) < 0.85)
             | orc.F_NO_FRUSTUM_CULLING * (rng.random(n) < 0.05) | orc.F_HAS_VIS_RANGE * (rng.random(n) < 0.3)
             | orc.F_NO_CPU_CULLING * (rng.random(n) < 0.05)).astype(np.uint8)
    return dict(rng=rng, n=n, gt=gt, bounds=bounds, flags=flags, caster=(rng.random(n) < 0.8).astype(np.uint8),
                layers=rng.integers(1, 4, n).astype(np.uint64), range_mask=rng.integers(0, 4, n).astype(np.uint32),
                bits=rng.permutation(n).astype(np.uint64) + 100, vv0=rng.choice([0, 2], n).astype(np.uint8))


def _gate(w, r, light_layers, range_bit):
    f = int(w["flags"][r])
    if not w["caster"][r] or f & orc.F_NO_CPU_CULLING or not f & orc.F_INHERITED_VISIBLE:
        return False
    if not int(light_layers) & int(w["layers"][r]):
        return False
    if f & orc.F_HAS_VIS_RANGE and (range_bit < 0 or not (w["range_mask"][r] >> range_bit) & 1):
        return False
    return True


def test_n3_spot_light_half_against_a_plain_loop():
    w = _shadow_world(21)
    rng, n = w["rng"], w["n"]
    L = 4
    lpos = rng.uniform(-15, 15, (L, 3)).astype(np.float32); lrange = rng.uniform(10, 35, L).astype(np.float32)
    llayers = rng.integers(1, 4, L).astype(np.uint64)
    ident = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1], np.float32)
    frusta = np.stack([orc.point_light_frusta(np.concatenate([ident, lpos[l]]), lrange[l], 0.1)[l % 6] for l in range(L)])
    vv, ch = w["vv0"].copy(), np.zeros(n, np.uint8)
    got = orc.check_spot_light_mesh_visibility(w["gt"], w["bounds"], w["flags"], w["caster"], w["bits"], vv, ch,
                                               np.concatenate([lpos, lrange[:, None]], 1), frusta, layer_mask=w["layers"],
                                               range_mask=w["range_mask"], lod_origin_index=0, light_layers=llayers)
    seen = np.zeros(n, bool)
    for l in range(L):
        rows = []
        for r in range(n):
            if not _gate(w, r, llayers[l], 0):
                continue
            f = int(w["flags"][r])
            if f & orc.F_HAS_AABB and not f & orc.F_NO_FRUSTUM_CULLING:
                b = w["bounds"][r]
                if not orc.sphere_intersects_obb(lpos[l], lrange[l], b[:3], b[3:], w["gt"][r]):
                    continue
                if not orc.intersects_obb(frusta[l], b[:3], b[3:], w["gt"][r], True, True):
                    continue
            rows.append(r); seen[r] = True
        assert np.array_equal(got[l], np.array(sorted(rows, key=lambda r: w["bits"][r]), np.uint32))
    assert seen.sum() > 20 and np.array_equal((vv & 1) != 0, seen) and np.array_equal(ch != 0, seen & (w["vv0"] == 0))


def test_n3_directional_light_half_against_a_plain_loop():
    w = _shadow_world(22)
    rng, n = w["rng"], w["n"]
    ident = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1], np.float32)

    def cascade(center, r):   # any six half spaces will do: reuse a cubemap face
        return orc.point_light_frusta(np.concatenate([ident, center]).astype(np.float32), r, 0.1)[int(rng.integers(0, 6))]
    items = [(np.stack([cascade(rng.uniform(-10, 10, 3), rr) for rr in (15.0, 30.0, 60.0)]), 3, 1),
             (np.stack([cascade(rng.uniform(-10, 10, 3), rr) for rr in (20.0, 50.0)]), 1, -1)]
    vv, ch = w["vv0"].copy(), np.zeros(n, np.uint8)
    got = orc.check_dir_light_mesh_visibility(w["gt"], w["bounds"], w["flags"], w["caster"], w["bits"], vv, ch, items,
                                              layer_mask=w["layers"], range_mask=w["range_mask"])
    seen = np.zeros(n, bool)
    for (fr, ll, vri), lists in zip(items, got):
        for c in range(len(fr)):
            rows = []
            for r in range(n):
                if not _gate(w, r, ll, vri):
                    continue
                f = int(w["flags"][r])
                if f & orc.F_HAS_AABB and not f & orc.F_NO_FRUSTUM_CULLING:
                    b = w["bounds"][r]
                    if not orc.intersects_obb(fr[c], b[:3], b[3:], w["gt"][r], False, True):   # near plane not tested
                        continue
                rows.append(r); seen[r] = True
            assert np.array_equal(lists[c], np.array(sorted(rows, key=lambda r: w["bits"][r]), np.uint32))
    assert seen.sum() > 20 and np.array_equal((vv & 1) != 0, seen) and np.array_equal(ch != 0, seen & (w["vv0"] == 0))
