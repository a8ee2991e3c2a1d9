"""CPU: GCN-Align adjacency / attribute-feature builders value-for-value against the reference's own GCN_Utils
and load_attr source (extracted; its results recorded under tests/golden) and against hand-computed cases."""
import numpy as np
import pytest
import scipy.sparse as sp

from oracle import gnn as orc_gnn
from tests.helpers import ReferenceRecording


def _gcn_utils():
    utils = orc_gnn.reference_gcn_utils()
    if utils is None:
        return None
    Utils, load_attr = utils
    return {"get_weighted_adj": lambda n, t: Utils(None, None).get_weighted_adj(n, t), "normalize_adj": Utils.normalize_adj,
            "load_attr": load_attr}


def _toy():
    # r=0: 3 triples, heads {0,1} tails {2,3} ; r=1: 1 triple ; one self loop that must be skipped
    return [(0, 0, 2), (0, 0, 3), (1, 0, 2), (2, 1, 3), (3, 1, 3)]


def test_weighted_adjacency_hand_computed():
    from openea_b200 import gnn
    tri = _toy()
    r2f, r2if = gnn.relation_functionality(tri)
    assert r2f[0] == pytest.approx(2 / 3) and r2if[0] == pytest.approx(2 / 3)
    assert r2f[1] == pytest.approx(2 / 2) and r2if[1] == pytest.approx(1 / 2)
    adj = gnn.weighted_adjacency(4, tri).toarray()
    # key (h,t) → entry [t, h] = max(r2if, .3) ; key (t,h) → entry [h, t] = max(r2f, .3)
    want = np.zeros((4, 4))
    for h, r, t in tri:
        if h == t:
            continue
        want[t, h] += max(r2if[r], 0.3)
        want[h, t] += max(r2f[r], 0.3)
    np.testing.assert_allclose(adj, want)
    norm = gnn.preprocess_adj(sp.csr_matrix(adj)).toarray()
    x = adj + np.eye(4)
    dis = 1 / np.sqrt(x.sum(1))
    np.testing.assert_allclose(norm, dis[:, None] * x.T * dis[None, :], rtol=1e-12)


def test_builders_equal_reference_source():
    from openea_b200 import gnn
    from openea_b200.synth import synth_id_arrays
    ref = ReferenceRecording("reference_gcn_builders", _gcn_utils)
    arr = synth_id_arrays("tiny", swapping=False)
    triples = [tuple(x) for x in np.concatenate([arr["triples1"], arr["triples2"]]).tolist()]
    n = arr["n_ent"]
    ref_adj = ref("get_weighted_adj", n, triples)
    mine = gnn.weighted_adjacency(n, triples)
    assert abs(sp.csr_matrix(ref_adj) - mine).max() < 1e-12
    ref_norm = ref("normalize_adj", ref_adj + sp.eye(n))
    assert abs(sp.csr_matrix(ref_norm) - sp.csr_matrix(gnn.preprocess_adj(mine))).max() < 1e-12
    rng = np.random.default_rng(0)
    ent_attrs = {int(e): set(rng.integers(0, 30, size=rng.integers(1, 5)).tolist()) for e in range(n)}

    class K:  # the two attributes of `kgs` load_attr reads
        pass
    kgs = K(); kgs.kg1 = K(); kgs.kg2 = K()
    kgs.kg1.entity_attributes_dict = {e: v for e, v in ent_attrs.items() if e % 2 == 0}
    kgs.kg2.entity_attributes_dict = {e: v for e, v in ent_attrs.items() if e % 2 == 1}
    ref_attr = ref("load_attr", n, kgs)
    mine_attr = gnn.attribute_features(n, {**kgs.kg1.entity_attributes_dict, **kgs.kg2.entity_attributes_dict})
    np.testing.assert_array_equal(ref_attr, mine_attr.toarray())
    ref.save()


def test_alinet_builders_equal_reference_source():
    """AKG / enhance_triples / no_weighted_adj / generate_2hop_triples / remove_unlinked_triples / generate_rel_ht of
    openea_b200.approaches.alinet against the reference's own source on a synthetic KG pair."""
    import contextlib
    import io
    from openea_b200.approaches import alinet as mine
    from openea_b200.synth import synth_id_arrays
    ref = ReferenceRecording("reference_alinet_builders", orc_gnn.reference_alinet_builders)
    arr = synth_id_arrays("tiny", swapping=False)
    t1 = {tuple(x) for x in arr["triples1"].tolist()}
    t2 = {tuple(x) for x in arr["triples2"].tolist()}
    with contextlib.redirect_stdout(io.StringIO()):
        mk1, mk2 = mine.AKG(t1), mine.AKG(t2)
    rk1, rk2 = ref("AKG", t1), ref("AKG", t2)
    assert mk1.out_related_ents_dict == rk1.out_related_ents_dict and mk1.in_related_ents_dict == rk1.in_related_ents_dict
    assert mk1.rt_dict == rk1.rt_dict and mk1.hr_dict == rk1.hr_dict and mk1.ent_list == rk1.ent_list
    sup1, sup2 = arr["train_links"][:, 0].tolist(), arr["train_links"][:, 1].tolist()
    linked = set(np.concatenate([arr["train_links"], arr["valid_links"], arr["test_links"]]).reshape(-1).tolist())
    with contextlib.redirect_stdout(io.StringIO()):
        me1, me2 = mine.enhance_triples(mk1, mk2, sup1, sup2)
        m_tri = mine.remove_unlinked_triples(mk1.triple_list + mk2.triple_list + list(me1) + list(me2), linked)
        m_adj, _ = mine.no_weighted_adj(arr["n_ent"], m_tri)
        m_two = mine.generate_2hop_triples(mk1, linked)
    re1, re2 = ref("enhance_triples", rk1, rk2, sup1, sup2)
    assert me1 == re1 and me2 == re2
    r_tri = ref("remove_unlinked_triples", rk1.triple_list + rk2.triple_list + sorted(re1) + sorted(re2), linked)
    assert set(m_tri) == set(r_tri)
    assert mine.generate_rel_ht(sorted(m_tri)) == ref("generate_rel_ht", sorted(r_tri))
    r_adj, _ = ref("no_weighted_adj", arr["n_ent"], r_tri, is_two_adj=False)
    coords, vals, shape = r_adj
    r_mat = sp.coo_matrix((vals, (coords[:, 0], coords[:, 1])), shape=shape).tocsr()
    assert abs(r_mat - sp.csr_matrix(m_adj)).max() < 1e-12
    r_two = ref("generate_2hop_triples", rk1, linked_ents=linked)
    # the 5 skipped patterns depend on tie order among equally frequent patterns: compare the path sets modulo that
    assert len(m_two ^ r_two) <= 0.05 * max(1, len(r_two)) or {(h, t) for h, _, t in m_two} == {(h, t) for h, _, t in r_two}
    ref.save()


def test_rdgcn_builders_equal_reference_source():
    """get_mat (degree quirk included) / rfunc / get_dual_input's Jaccard matrix against the reference's own source."""
    import math
    from openea_b200.approaches import rdgcn as mine
    from openea_b200.synth import synth_id_arrays
    ref = ReferenceRecording("reference_rdgcn_builders", orc_gnn.reference_rdgcn_builders)
    arr = synth_id_arrays("tiny", swapping=False)
    triples = [tuple(x) for x in np.concatenate([arr["triples1"], arr["triples2"]]).tolist()]
    E, R = arr["n_ent"], arr["n_rel"]
    pos, degree = ref("get_mat", triples, E)
    M = mine.get_sparse_matrix(triples, E).todok()
    assert len(M) == len(pos)
    for (fir, sec), v in list(pos.items())[::37]:
        assert M[sec, fir] == pytest.approx(v / math.sqrt(degree[fir]) / math.sqrt(degree[sec]), rel=1e-12)
    _, mdeg = mine.get_mat(triples, E)
    assert mdeg.tolist() == list(degree)
    head, tail, head_r, tail_r, r_mat = ref("rfunc", triples, E, R)
    mh, mt, tri = mine.rfunc(triples, E, R)
    np.testing.assert_array_equal(mh.toarray(), head_r.T)
    np.testing.assert_array_equal(mt.toarray(), tail_r.T)
    assert sorted(map(tuple, np.stack([tri[:, 0], tri[:, 2], tri[:, 1]], 1).tolist())) == \
        sorted((i[0], i[1], v) for i, v in zip(r_mat[0], r_mat[1]))
    dual = mine.dual_adjacency(mh, mt)
    for i, j in ((0, 0), (0, 1), (3, 7), (R - 1, 2)):
        want = len(head[i] & head[j]) / len(head[i] | head[j]) + len(tail[i] & tail[j]) / len(tail[i] | tail[j])
        assert dual[i, j] == pytest.approx(want, rel=1e-6)
    ref.save()


def test_graph_builders_give_the_same_graphs_from_either_dataset_loader(tmp_path, monkeypatch):
    """The adjacency / incidence builders of GCN-Align, AliNet and RDGCN consume the KG containers
    (`relation_triples_list`, `relation_triples_set`, `entity_attributes_dict`, link lists); they must build identical
    matrices from the array-backed loader (sorted, lazily built containers) and from the container-based loader."""
    import contextlib
    import io
    import scipy.sparse as sp
    from openea_b200 import gnn
    from openea_b200.approaches import alinet, rdgcn
    from openea_b200.modules.load.kgs import read_kgs_from_folder
    from openea_b200.modules.utils.util import merge_dic
    from openea_b200.synth import write_dataset
    folder = write_dataset(str(tmp_path) + "/tiny/", "tiny")
    monkeypatch.setenv("OEA_NO_DATASET_CACHE", "1")
    built = {}
    for loader in ("arrays", "containers"):
        monkeypatch.setenv("OEA_LOADER", loader)
        with contextlib.redirect_stdout(io.StringIO()):
            kgs = read_kgs_from_folder(folder, "721_5fold/1/", "mapping", True)
            n = kgs.entities_num
            triples = kgs.kg1.relation_triples_list + kgs.kg2.relation_triples_list
            out = {"gcn_adj": gnn.preprocess_adj(gnn.weighted_adjacency(n, triples)),
                   "gcn_attr": gnn.attribute_features(n, merge_dic(kgs.kg1.entity_attributes_dict,
                                                                   kgs.kg2.entity_attributes_dict))}
            kg1, kg2 = alinet.AKG(kgs.kg1.relation_triples_set), alinet.AKG(kgs.kg2.relation_triples_set)
            linked = set(kgs.train_entities1 + kgs.train_entities2 + kgs.valid_entities1 + kgs.test_entities1 +
                         kgs.test_entities2 + kgs.valid_entities2)
            enh1, enh2 = alinet.enhance_triples(kg1, kg2, kgs.train_entities1, kgs.train_entities2)
            tri = alinet.remove_unlinked_triples(kg1.triple_list + kg2.triple_list + list(enh1) + list(enh2), linked)
            out["alinet_one"] = alinet.no_weighted_adj(n, tri)[0]
            two = alinet.generate_2hop_triples(kg1, linked) | alinet.generate_2hop_triples(kg2, linked)
            out["alinet_two"] = alinet.no_weighted_adj(n, list(two))[0]
            out["alinet_rel_ht"] = {r: (sorted(v[0]), sorted(v[1])) if isinstance(v, tuple) else sorted(v)
                                    for r, v in alinet.generate_rel_ht(tri).items()}
            out["rdgcn_M"] = rdgcn.get_sparse_matrix(triples, n)
            head_r, tail_r, _ = rdgcn.rfunc(triples, n, kgs.relations_num)
            out["rdgcn_head_r"], out["rdgcn_tail_r"] = head_r, tail_r
        built[loader] = out
    a, b = built["arrays"], built["containers"]
    assert a.keys() == b.keys()
    for name in a:
        x, y = a[name], b[name]
        if name == "alinet_rel_ht":
            assert x == y
            continue
        if name == "gcn_attr":
            # load_attr ranks attributes by frequency with ties in dict / set iteration order (string hashes differ
            # per process, in the reference too): compare the columns as a multiset, leaving out the least frequent
            # ones, where a tie at the 70 % cut-off may select different attributes
            def columns(m):
                m = sp.csc_matrix(m)
                cols = [tuple(m.indices[m.indptr[j]:m.indptr[j + 1]].tolist()) for j in range(m.shape[1])]
                cut = min(len(c) for c in cols)
                return sorted(c for c in cols if len(c) > cut)
            assert x.shape == y.shape and columns(x) == columns(y)
            continue
        if isinstance(x, tuple):         # sparse_to_tuple form: (coords, values, shape)
            x, y = sp.coo_matrix((x[1], (x[0][:, 0], x[0][:, 1])), shape=x[2]), sp.coo_matrix((y[1], (y[0][:, 0], y[0][:, 1])), shape=y[2])
        x, y = sp.csr_matrix(x), sp.csr_matrix(y)
        assert x.shape == y.shape and abs(x - y).max() < 1e-6, name


@pytest.mark.parametrize("seed", range(6))
def test_alinet_array_builders_equal_the_set_based_builders(seed):
    """approaches/alinet_graph.py (sorted-key joins on arrays) against the set / dict builders of approaches/alinet.py,
    which are themselves pinned to the reference's source above: enhanced triples, two-hop pairs (the 5 most frequent
    relation patterns dropped), both adjacencies, the relation index."""
    import contextlib
    import io
    from openea_b200.approaches import alinet, alinet_graph as ag
    rng = np.random.default_rng(seed)
    n, n_rel = 90, 7

    def kg(lo, hi, m):
        hub = rng.integers(lo, lo + 6, m)                                   # a few hubs: many two-hop paths
        t = np.stack([np.where(rng.random(m) < 0.3, hub, rng.integers(lo, hi, m)), rng.integers(0, n_rel, m),
                      rng.integers(lo, hi, m)], 1)
        return np.unique(t, axis=0)
    t1, t2 = kg(0, 45, 160), kg(45, 90, 150)
    sup1, sup2 = rng.permutation(45)[:12], 45 + rng.permutation(45)[:12]
    linked = set(rng.permutation(n)[:70].tolist()) | set(sup1.tolist()) | set(sup2.tolist())
    with contextlib.redirect_stdout(io.StringIO()):
        k1, k2 = alinet.AKG([tuple(x) for x in t1.tolist()]), alinet.AKG([tuple(x) for x in t2.tolist()])
        want_new1, want_new2 = alinet.enhance_triples(k1, k2, sup1.tolist(), sup2.tolist())
        got_new1, got_new2 = ag.enhance(t1, t2, sup1, sup2, n)
        assert {tuple(x) for x in got_new1.tolist()} == want_new1 and {tuple(x) for x in got_new2.tolist()} == want_new2
        for kg_obj, tri in ((k1, t1), (k2, t2)):
            # the reference orders equally frequent patterns by set iteration order: only compare when rank 5 / 6 differ
            pats = {}
            by_head = {}
            lt = alinet.remove_unlinked_triples(kg_obj.triples, linked)
            for h, r, t in lt:
                by_head.setdefault(h, []).append((r, t))
            for h, rx, m in lt:
                for ry, t in by_head.get(m, ()):
                    if (h, t) not in kg_obj.ht:
                        pats[(rx, ry)] = pats.get((rx, ry), 0) + 1
            counts = sorted(pats.values(), reverse=True)
            got = {tuple(x) for x in ag.two_hop_pairs(tri, linked, n, chunk=97).tolist()}     # tiny chunks: many of them
            # the same selection with the array version's documented tie order (count desc, then (r_x, r_y))
            dropped = {p for p, _ in sorted(pats.items(), key=lambda kv: (-kv[1], kv[0]))[:5]}
            want = set()
            for h, rx, m in lt:
                for ry, t in by_head.get(m, ()):
                    if (h, t) not in kg_obj.ht and (rx, ry) not in dropped:
                        want.update([(h, t), (h, h)])
            assert got == want and len(got) > 0
            if len(counts) <= 5 or counts[4] != counts[5]:                   # no tie at the cut: the pinned builder agrees too
                assert got == {(h, t) for h, _, t in alinet.generate_2hop_triples(kg_obj, linked)}
        tri_all = alinet.remove_unlinked_triples(k1.triple_list + k2.triple_list + list(want_new1) + list(want_new2), linked)
        want_one = alinet.no_weighted_adj(n, tri_all)[0]
        one, two, tri = ag.build(t1, t2, sup1, sup2, linked, n)
        assert {tuple(x) for x in tri.tolist()} == set(tri_all)
        assert abs(sp.csr_matrix(one) - sp.csr_matrix(want_one)).max() < 1e-12
        rels, ptr, pairs = ag.relation_index(tri)
        want_ht = alinet.generate_rel_ht(tri_all)
        assert sorted(rels.tolist()) == sorted(want_ht)
        for i, r in enumerate(rels.tolist()):
            assert sorted(map(tuple, pairs[ptr[i]:ptr[i + 1]].tolist())) == sorted(want_ht[r])
