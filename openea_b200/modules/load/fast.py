"""Array-backed dataset layer (SURVEY §8f-3): the reference's TSV readers, id assignment and KG / KGs containers
(modules/load/{read,kg,kgs}.py) with NumPy arrays as the primary representation and a binary cache.

Why: at the 100K shape the reference-style loader spends 20–30 s building Python sets / dicts of 1–2 million tuples for
four KG objects before the first training step, while a training epoch on the GPU takes milliseconds.  Here

  * the TSV files are parsed by the pandas C reader, rows de-duplicated and strings interned with vectorised
    factorisation; ids are assigned exactly as `sort_elements` / `generate_mapping_id` / `generate_sharing_id`
    (read.py:12-92) do for `ordered=True` — by (occurrence count, name) descending, the two KGs interleaved;
  * a KG is three int32 arrays (relation triples, attribute triples with an interned value column, vocabularies);
    every attribute name of the reference's `KG` (`relation_triples_set`, `rt_dict`, `entities_list`, … kg.py:10-141) is
    still there but is built on first access (`ArrayKG.__getattr__`), so code that never asks for a Python container
    never pays for it; the device layer takes `relation_triples_array` without a copy;
  * swap ("supervised") triples of the 'swapping' mode (read.py:136-167, kgs.py:45-50) are generated with array ops;
  * the finished arrays are cached in one .npz keyed by the input files' sizes / mtimes and the load arguments
    (`$OEA_CACHE_DIR`, default ~/.cache/openea_b200); a cached load does no parsing at all.

Anything this path does not cover exactly (unordered ids — they depend on Python set iteration order —, RSN4EA's
`remove_unlinked`, the DBP15K / DWY100K layouts, attribute lines that need the reference's multi-tab value joining)
falls back to the container-based loader in kgs.py, which mirrors the reference line by line.
tests/test_host_modules.py compares both loaders with the reference's recorded results in all three id modes.
"""
import csv
import hashlib
import os
import time

import numpy as np

CACHE_VERSION = 4


class Unsupported(Exception):
    """This dataset / argument combination needs the container-based loader."""


# ---- parsing ---------------------------------------------------------------------------------------------------------
def _tabs_per_line(path):
    """Number of tab characters on every line of a file (vectorised over the raw bytes)."""
    with open(path, "rb") as fh:
        buf = np.frombuffer(fh.read(), dtype=np.uint8)
    if buf.size == 0:
        return np.zeros(0, dtype=np.int64)
    ends = np.flatnonzero(buf == 10)
    if ends.size == 0 or ends[-1] != buf.size - 1:
        ends = np.append(ends, buf.size - 1)                  # last line without a newline
    tabs_before = np.searchsorted(np.flatnonzero(buf == 9), ends, side="right")
    return np.diff(tabs_before, prepend=0)


def _read_tsv(path, n_cols, tabs=None):
    """Columns of a TSV file as object arrays of stripped strings (read.py:222-257 strip every field).  Every line must
    hold exactly n_cols fields (the reference asserts it); anything else is left to the container-based reader."""
    import pandas as pd
    tabs = _tabs_per_line(path) if tabs is None else tabs
    if tabs.size == 0:
        return [np.zeros(0, dtype=object) for _ in range(n_cols)]
    if (tabs != n_cols - 1).any():
        raise Unsupported("%s: a line does not have %d tab-separated fields" % (path, n_cols))
    try:
        df = pd.read_csv(path, sep="\t", header=None, names=list(range(n_cols)), index_col=False, dtype=str,
                         quoting=csv.QUOTE_NONE, na_filter=False, encoding="utf8", engine="c", skip_blank_lines=False)
    except (pd.errors.ParserError, ValueError) as e:
        raise Unsupported("%s: %s" % (path, e))
    if len(df) != tabs.size:
        raise Unsupported("%s: line count mismatch" % path)
    return [df[i].str.strip().to_numpy(dtype=object) for i in range(n_cols)]


def _read_relation_triples(path):
    return _read_tsv(path, 3)


def _read_attribute_triples(path):
    """read.py:239-257: lines with fewer than three fields are skipped; the value loses surrounding blanks and a
    trailing '.'; extra tab-separated pieces are joined into the value (left to the container-based reader)."""
    import pandas as pd
    tabs = _tabs_per_line(path)
    if (tabs > 2).any() or (tabs < 2).any():
        raise Unsupported("%s: attribute lines that need the reference's skipping / value joining" % path)
    e, a, v = _read_tsv(path, 3, tabs)
    v = pd.Series(v, dtype=object).str.strip().str.rstrip(".").str.strip().to_numpy(dtype=object)
    return e, a, v


def _read_links(path):
    a, b = _read_tsv(path, 2)
    return a, b


def _unique_rows(*cols):
    """De-duplicated rows (the reference keeps triples in a set) → tuple of arrays, first-seen order."""
    import pandas as pd
    if len(cols[0]) == 0:
        return cols
    df = pd.DataFrame({i: c for i, c in enumerate(cols)})
    df = df.drop_duplicates(ignore_index=True)
    return tuple(df[i].to_numpy() for i in range(len(cols)))


# ---- id assignment (read.py:12-92) -------------------------------------------------------------------------------------
def _ordered_elements(names, triple_cols):
    """`names` (unique strings) ordered by (occurrences in the three triple columns, name) descending: sort_elements."""
    import pandas as pd
    index = pd.Index(names)
    counts = np.zeros(len(names), dtype=np.int64)
    for col in triple_cols:
        pos = index.get_indexer(col)
        counts += np.bincount(pos[pos >= 0], minlength=len(names))
    name_rank = np.empty(len(names), dtype=np.int64)
    name_rank[np.argsort(np.asarray(names, dtype=str), kind="stable")] = np.arange(len(names))
    order = np.lexsort((name_rank, counts))[::-1]            # ascending by (count, name) → reversed
    return order


def _mapping_ids(names1, cols1, names2, cols2):
    """generate_mapping_id(ordered=True): rank i of KG1 → 2i, of KG2 → 2i+1; the longer list's overflow follows."""
    o1, o2 = _ordered_elements(names1, cols1), _ordered_elements(names2, cols2)
    n1, n2 = len(o1), len(o2)
    both = min(n1, n2)
    ids1, ids2 = np.empty(n1, dtype=np.int64), np.empty(n2, dtype=np.int64)
    ids1[o1[:both]] = 2 * np.arange(both)
    ids2[o2[:both]] = 2 * np.arange(both) + 1
    ids1[o1[both:]] = 2 * n2 + (np.arange(both, n1) - n2)
    ids2[o2[both:]] = 2 * n1 + (np.arange(both, n2) - n1)
    return ids1, ids2


def _sharing_ids(names1, cols1, names2, cols2, links):
    """generate_sharing_id(ordered=True): seed-linked KG2 elements reuse their KG1 counterpart's id; the others get
    mapping ids computed WITHOUT the linked elements (read.py:36-43)."""
    import pandas as pd
    l1, l2 = links
    if len(l1) == 0:
        return _mapping_ids(names1, cols1, names2, cols2)
    idx1, idx2 = pd.Index(names1), pd.Index(names2)
    linked2 = idx2.get_indexer(l2)
    if (linked2 < 0).any() or (idx1.get_indexer(l1) < 0).any():
        raise Unsupported("a train link names an entity without triples")     # the reference raises KeyError there
    counterpart = {}
    for x, y in zip(l1, l2):                                   # {y: x for x, y in train_links}: the last x wins
        counterpart[y] = x
    unlinked_mask = np.ones(len(names2), dtype=bool)
    unlinked_mask[linked2] = False
    ids1, ids2_unlinked = _mapping_ids(names1, cols1, names2[unlinked_mask], cols2)
    ids2 = np.empty(len(names2), dtype=np.int64)
    ids2[unlinked_mask] = ids2_unlinked
    ys = np.array(list(counterpart.keys()), dtype=object)
    xs = np.array(list(counterpart.values()), dtype=object)
    ids2[idx2.get_indexer(ys)] = ids1[idx1.get_indexer(xs)]
    return ids1, ids2


# ---- containers ----------------------------------------------------------------------------------------------------------
def _group_pairs(keys, vals):
    out = {}
    for k, v in zip(keys, vals):
        out.setdefault(k, set()).add(v)
    return out


class ArrayKG:
    """Duck type of modules/load/kg.KG over arrays.  `ent`, `rel`, `attr`, `val` are decoders: None for id KGs (the array
    entries ARE the reference's values) or object arrays of strings for URI-level KGs.  Values of attribute triples are
    always strings (`val` vocabulary).

    Laziness contract: the `*_array` / `*_num` attributes are plain members; every other attribute name of the
    reference's KG is produced by `_BUILDERS` on first access and then stored on the instance."""

    def __init__(self, rel_triples, attr_triples, values, ent=None, rel=None, attr=None):
        self.relation_triples_array = self.local_relation_triples_array = np.ascontiguousarray(rel_triples, dtype=np.int32).reshape(-1, 3)
        self.attribute_triples_array = self.local_attribute_triples_array = np.ascontiguousarray(attr_triples, dtype=np.int32).reshape(-1, 3)
        self.values, self._ent, self._rel, self._attr = values, ent, rel, attr
        self.sup_relation_triples_array = self.sup_attribute_triples_array = None
        r, a = self.relation_triples_array, self.attribute_triples_array
        self.entities_array = np.unique(np.concatenate([r[:, 0], r[:, 2], a[:, 0]]))
        self.relations_array = np.unique(r[:, 1])
        self.attributes_array = np.unique(a[:, 1])
        self.entities_num, self.relations_num = len(self.entities_array), len(self.relations_array)
        self.attributes_num = len(self.attributes_array)
        self.relation_triples_num = self.local_relation_triples_num = len(r)
        self.attribute_triples_num = self.local_attribute_triples_num = len(a)
        self._id_sources = {}      # 'entities' / 'relations' / 'attributes' → (names, ids); dicts are built on first read

    # -- decoding ----------------------------------------------------------------------------------------------
    def _dec(self, ids, table):
        return ids.tolist() if table is None else table[ids].tolist()

    def _rel_tuples(self, arr):
        return list(zip(self._dec(arr[:, 0], self._ent), self._dec(arr[:, 1], self._rel), self._dec(arr[:, 2], self._ent)))

    def _attr_tuples(self, arr):
        return list(zip(self._dec(arr[:, 0], self._ent), self._dec(arr[:, 1], self._attr), self.values[arr[:, 2]].tolist()))

    # -- lazy reference attributes ---------------------------------------------------------------------------------
    def _build_relation_sets(self):
        local = self._rel_tuples(self.local_relation_triples_array)
        merged = local if self.sup_relation_triples_array is None else self._rel_tuples(self.relation_triples_array)
        tset = set(merged)
        # kg.py: `relation_triples_set` and `local_relation_triples_set` are ONE object, so the in-place merge of the
        # swap triples (add_sup_relation_triples) shows in both; the local LIST keeps the pre-merge triples
        self.relation_triples_set = self.local_relation_triples_set = tset
        self.relation_triples_list = merged
        self.local_relation_triples_list = local

    def _build_attribute_sets(self):
        local = self._attr_tuples(self.local_attribute_triples_array)
        merged = local if self.sup_attribute_triples_array is None else self._attr_tuples(self.attribute_triples_array)
        self.attribute_triples_set = self.local_attribute_triples_set = set(merged)
        self.attribute_triples_list = merged
        self.local_attribute_triples_list = local

    def _build_vocab(self, name, arr, table):
        items = self._dec(arr, table)
        setattr(self, name + "_set", set(items))
        setattr(self, name + "_list", items)

    def _build_relation_dicts(self):
        local = self.local_relation_triples_list
        self.rt_dict = _group_pairs((h for h, _, _ in local), ((r, t) for _, r, t in local))
        self.hr_dict = _group_pairs((t for _, _, t in local), ((h, r) for h, r, _ in local))
        # parse_relations reads local_relation_triples_SET, which is built before any swap triples are merged
        self.entity_relations_dict = _group_pairs((h for h, _, _ in local), (r for _, r, _ in local))

    def _build_attribute_dicts(self):
        local = self.local_attribute_triples_list
        self.av_dict = _group_pairs((e for e, _, _ in local), ((a, v) for _, a, v in local))
        self.entity_attributes_dict = _group_pairs((e for e, _, _ in local), (a for _, a, _ in local))

    # reference attribute name → the method that materialises it (together with its siblings) on first access
    _BUILDERS = dict(
        [(n, "_build_relation_sets") for n in ("relation_triples_set", "relation_triples_list",
                                               "local_relation_triples_set", "local_relation_triples_list")] +
        [(n, "_build_attribute_sets") for n in ("attribute_triples_set", "attribute_triples_list",
                                                "local_attribute_triples_set", "local_attribute_triples_list")] +
        [(n, "_build_relation_dicts") for n in ("rt_dict", "hr_dict", "entity_relations_dict")] +
        [(n, "_build_attribute_dicts") for n in ("av_dict", "entity_attributes_dict")])

    def __getattr__(self, name):                 # only reached when the attribute is not on the instance yet
        for kind in ("relation", "attribute"):
            if name in ("sup_%s_triples_set" % kind, "sup_%s_triples_list" % kind) and "values" in self.__dict__:
                self._build_sup(kind)
                return self.__dict__[name]
        fn = ArrayKG._BUILDERS.get(name)
        if fn is not None:
            getattr(self, fn)()
            return self.__dict__[name]
        for vocab, arr, table in (("entities", "entities_array", "_ent"), ("relations", "relations_array", "_rel"),
                                  ("attributes", "attributes_array", "_attr")):
            if name in (vocab + "_set", vocab + "_list"):
                self._build_vocab(vocab, self.__dict__[arr], self.__dict__[table])
                return self.__dict__[name]
            if name == vocab + "_id_dict" and "_id_sources" in self.__dict__:
                src = self._id_sources.get(vocab)
                value = None if src is None else dict(zip(src[0].tolist(), src[1].tolist()))
                self.__dict__[name] = value
                return value
        raise AttributeError(name)

    # -- reference API ------------------------------------------------------------------------------------------------
    def set_id_dict(self, entities_id_dict, relations_id_dict, attributes_id_dict):
        self.entities_id_dict, self.relations_id_dict, self.attributes_id_dict = \
            entities_id_dict, relations_id_dict, attributes_id_dict

    def set_id_sources(self, entities, relations, attributes):
        """(names, ids) array pairs from which the {uri: id} dicts of set_id_dict are built when first read
        (read.py:325-349 writes them at the end of a run)."""
        self._id_sources = dict(entities=entities, relations=relations, attributes=attributes)

    def _set_sup(self, kind, sup_unique, merged):
        """Install de-duplicated swap triples and the merged (local ∪ swap) triples of one kind."""
        setattr(self, "sup_%s_triples_array" % kind, sup_unique)
        setattr(self, "%s_triples_array" % kind, merged)
        setattr(self, "%s_triples_num" % kind, len(merged))
        for n in ("%s_triples_set", "%s_triples_list", "local_%s_triples_set", "local_%s_triples_list",
                  "sup_%s_triples_set", "sup_%s_triples_list"):
            self.__dict__.pop(n % kind, None)     # (re)built lazily

    def _build_sup(self, kind):
        arr = getattr(self, "sup_%s_triples_array" % kind)
        tuples = None if arr is None else (self._rel_tuples(arr) if kind == "relation" else self._attr_tuples(arr))
        self.__dict__["sup_%s_triples_list" % kind] = tuples
        self.__dict__["sup_%s_triples_set" % kind] = None if tuples is None else set(tuples)

    def add_sup_relation_triples(self, sup_triples):
        """kg.py:126-133 with id tuples (or an [n, 3] array) as input."""
        sup = unique_int_rows(np.asarray(list(sup_triples) if isinstance(sup_triples, (set, frozenset)) else sup_triples,
                                         dtype=np.int32).reshape(-1, 3))
        self._set_sup("relation", sup, unique_int_rows(np.concatenate([self.relation_triples_array, sup])))

    def add_sup_attribute_triples(self, sup_triples):
        """[n, 3] int array (entity id, attribute id, value index in this KG's value vocabulary)."""
        sup = unique_int_rows(np.asarray(sup_triples, dtype=np.int32).reshape(-1, 3))
        self._set_sup("attribute", sup, unique_int_rows(np.concatenate([self.attribute_triples_array, sup])))


def unique_int_rows(arr):
    """Distinct rows of a non-negative int [n, 3] array (set semantics of the reference's triple containers)."""
    arr = np.ascontiguousarray(arr, dtype=np.int32).reshape(-1, 3)
    if len(arr) == 0:
        return arr
    bits = [int(arr[:, c].max()).bit_length() for c in range(3)]
    if sum(bits) <= 63:
        a = arr.astype(np.int64)
        key = (a[:, 0] << (bits[1] + bits[2])) | (a[:, 1] << bits[2]) | a[:, 2]
        _, first = np.unique(key, return_index=True)
        return arr[np.sort(first)]
    import pandas as pd
    return pd.DataFrame(arr).drop_duplicates().to_numpy(dtype=np.int32)


class ArrayKGs:
    """Duck type of modules/load/kgs.KGs (kgs.py:5-99) over ArrayKG."""

    def __init__(self, parts):
        p = parts
        self.kg1, self.kg2 = p["kg1"], p["kg2"]
        self.uri_kg1, self.uri_kg2 = p["uri_kg1"], p["uri_kg2"]
        for name in ("train", "test", "valid"):
            arr = p[name + "_links"]
            setattr(self, name + "_links_array", arr)
            setattr(self, name + "_links", list(zip(arr[:, 0].tolist(), arr[:, 1].tolist())))
            setattr(self, name + "_entities1", arr[:, 0].tolist())
            setattr(self, name + "_entities2", arr[:, 1].tolist())
            setattr(self, "uri_%s_links" % name, p["uri_%s_links" % name])
        self.useful_entities_list1 = self.kg1.entities_list
        self.useful_entities_list2 = self.kg2.entities_list
        self.entities_num = len(np.union1d(self.kg1.entities_array, self.kg2.entities_array))
        self.relations_num = len(np.union1d(self.kg1.relations_array, self.kg2.relations_array))
        self.attributes_num = len(np.union1d(self.kg1.attributes_array, self.kg2.attributes_array))


# ---- the loader ------------------------------------------------------------------------------------------------------------
def _intern(cols_by_vocab):
    """Factorise several string columns over ONE vocabulary → (codes per column, unique names as object array)."""
    import pandas as pd
    lens = [len(c) for c in cols_by_vocab]
    codes, names = pd.factorize(np.concatenate(cols_by_vocab) if lens else np.zeros(0, dtype=object))
    out, at = [], 0
    for n in lens:
        out.append(codes[at:at + n].astype(np.int64))
        at += n
    return out, np.asarray(names, dtype=object)


def _swap_triples(tri, link_from, link_to, n_ids):
    """generate_sup_relation_triples for one KG (read.py:136-148): for a link (e1 → e2) every triple with head e1 yields
    (e2, r, t) and every triple with tail e1 yields (h, r, e2) — one end per generated triple."""
    to = np.full(n_ids, -1, dtype=np.int64)
    to[link_from] = link_to
    hs, ts = to[tri[:, 0]], to[tri[:, 2]]
    a = tri[hs >= 0].copy()
    a[:, 0] = hs[hs >= 0]
    b = tri[ts >= 0].copy()
    b[:, 2] = ts[ts >= 0]
    return np.concatenate([a, b]) if len(a) + len(b) else np.zeros((0, 3), dtype=tri.dtype)


def _swap_attr_triples(tri, link_from, link_to, n_ids):
    to = np.full(n_ids, -1, dtype=np.int64)
    to[link_from] = link_to
    es = to[tri[:, 0]]
    a = tri[es >= 0].copy()
    a[:, 0] = es[es >= 0]
    return a


def build(folder, division, mode, ordered):
    """Parse + assign ids + assemble.  Returns the dict of primary arrays (what the cache stores)."""
    if not ordered:
        raise Unsupported("unordered ids follow Python set iteration order")
    raw = {}
    for side in ("1", "2"):
        raw["rel" + side] = _unique_rows(*_read_relation_triples(folder + "rel_triples_" + side))
        raw["attr" + side] = _unique_rows(*_read_attribute_triples(folder + "attr_triples_" + side))
    links = {name: _read_links(folder + division + name + "_links") for name in ("train", "valid", "test")}

    out = {}
    uri = {}
    for side in ("1", "2"):
        (h, r, t), (e, a, v) = raw["rel" + side], raw["attr" + side]
        (hc, tc, ec), ent_names = _intern([h, t, e])
        (rc,), rel_names = _intern([r])
        (ac,), attr_names = _intern([a])
        (vc,), val_names = _intern([v])
        uri[side] = dict(rel=np.stack([hc, rc, tc], 1) if len(hc) else np.zeros((0, 3), np.int64),
                         attr=np.stack([ec, ac, vc], 1) if len(ec) else np.zeros((0, 3), np.int64),
                         ent_names=ent_names, rel_names=rel_names, attr_names=attr_names, val_names=val_names,
                         rel_cols=(h, r, t), attr_cols=(e, a, v))
    u1, u2 = uri["1"], uri["2"]
    make = _sharing_ids if mode == "sharing" else (lambda n1, c1, n2, c2, links_: _mapping_ids(n1, c1, n2, c2))
    none = (np.zeros(0, dtype=object),) * 2
    ent_ids1, ent_ids2 = make(u1["ent_names"], u1["rel_cols"], u2["ent_names"], u2["rel_cols"], links["train"])
    rel_ids1, rel_ids2 = make(u1["rel_names"], u1["rel_cols"], u2["rel_names"], u2["rel_cols"], none)
    attr_ids1, attr_ids2 = make(u1["attr_names"], u1["attr_cols"], u2["attr_names"], u2["attr_cols"], none)

    import pandas as pd
    idx1, idx2 = pd.Index(u1["ent_names"]), pd.Index(u2["ent_names"])
    for name, (a, b) in links.items():
        pa, pb = idx1.get_indexer(a), idx2.get_indexer(b)
        ok = (pa >= 0) & (pb >= 0)                                         # uris_pair_2ids drops unknown entities
        out[name + "_links"] = np.stack([ent_ids1[pa[ok]], ent_ids2[pb[ok]]], 1).astype(np.int32).reshape(-1, 2)
        out["uri_%s_links_a" % name], out["uri_%s_links_b" % name] = np.asarray(a, dtype=str), np.asarray(b, dtype=str)

    for side, u, eid, rid, aid in (("1", u1, ent_ids1, rel_ids1, attr_ids1), ("2", u2, ent_ids2, rel_ids2, attr_ids2)):
        rel = np.stack([eid[u["rel"][:, 0]], rid[u["rel"][:, 1]], eid[u["rel"][:, 2]]], 1) if len(u["rel"]) else np.zeros((0, 3))
        attr = np.stack([eid[u["attr"][:, 0]], aid[u["attr"][:, 1]], u["attr"][:, 2]], 1) if len(u["attr"]) else np.zeros((0, 3))
        out["rel" + side], out["attr" + side] = rel.astype(np.int32), attr.astype(np.int32)
        out["uri_rel" + side], out["uri_attr" + side] = u["rel"].astype(np.int32), u["attr"].astype(np.int32)
        for k in ("ent_names", "rel_names", "attr_names", "val_names"):
            out[k + side] = np.asarray(u[k], dtype=str)            # fixed-width unicode: the cache holds no pickles
        out["ent_ids" + side], out["rel_ids" + side], out["attr_ids" + side] = eid, rid, aid

    if mode == "swapping":
        n_ids = int(max(ent_ids1.max(initial=-1), ent_ids2.max(initial=-1))) + 1
        tl = out["train_links"].astype(np.int64)
        out["sup_rel1"] = unique_int_rows(_swap_triples(out["rel1"], tl[:, 0], tl[:, 1], n_ids))
        out["sup_rel2"] = unique_int_rows(_swap_triples(out["rel2"], tl[:, 1], tl[:, 0], n_ids))
        # KG1's swap triples are KG1's own triples with the subject replaced by its KG2 counterpart (read.py:151-167), so
        # their attribute ids and value indices stay in KG1's vocabularies
        out["sup_attr1"] = unique_int_rows(_swap_attr_triples(out["attr1"], tl[:, 0], tl[:, 1], n_ids))
        out["sup_attr2"] = unique_int_rows(_swap_attr_triples(out["attr2"], tl[:, 1], tl[:, 0], n_ids))
        for side in ("1", "2"):           # merged = local ∪ swap (kg.py:126-133), stored so a cached load does no set work
            out["merged_rel" + side] = unique_int_rows(np.concatenate([out["rel" + side], out["sup_rel" + side]]))
            out["merged_attr" + side] = unique_int_rows(np.concatenate([out["attr" + side], out["sup_attr" + side]]))
    out["mode"] = np.array(mode)
    return out


def assemble(parts):
    """ArrayKGs from the primary arrays."""
    p = parts
    mode = str(p["mode"])
    kgs = {}
    for side in ("1", "2"):
        vals = p["val_names" + side]
        kg = ArrayKG(p["rel" + side], p["attr" + side], vals)
        kg.set_id_sources((p["ent_names" + side], p["ent_ids" + side]), (p["rel_names" + side], p["rel_ids" + side]),
                          (p["attr_names" + side], p["attr_ids" + side]))
        if mode == "swapping":
            kg._set_sup("relation", p["sup_rel" + side], p["merged_rel" + side])
            kg._set_sup("attribute", p["sup_attr" + side], p["merged_attr" + side])
        kgs["kg" + side] = kg
        kgs["uri_kg" + side] = ArrayKG(p["uri_rel" + side], p["uri_attr" + side], vals, ent=p["ent_names" + side],
                                       rel=p["rel_names" + side], attr=p["attr_names" + side])
    for name in ("train", "valid", "test"):
        kgs[name + "_links"] = p[name + "_links"]
        kgs["uri_%s_links" % name] = list(zip(np.asarray(p["uri_%s_links_a" % name]).tolist(),
                                              np.asarray(p["uri_%s_links_b" % name]).tolist()))
    return ArrayKGs(kgs)


# ---- binary cache ---------------------------------------------------------------------------------------------------------
def _signature(folder, division, mode, ordered):
    h = hashlib.sha1()
    h.update(repr((CACHE_VERSION, os.path.abspath(folder), division, mode, bool(ordered))).encode())
    for rel in ["rel_triples_1", "rel_triples_2", "attr_triples_1", "attr_triples_2"] + \
               [division + n + "_links" for n in ("train", "valid", "test")]:
        st = os.stat(folder + rel)
        h.update(repr((rel, st.st_size, st.st_mtime_ns)).encode())
    return h.hexdigest()


def cache_dir():
    return os.environ.get("OEA_CACHE_DIR") or os.path.join(os.path.expanduser("~"), ".cache", "openea_b200")


def load(folder, division, mode, ordered, remove_unlinked=False, use_cache=True, verbose=True):
    """ArrayKGs of a dataset folder in the reference's layout; raises Unsupported for what only kgs.py covers."""
    lowered = folder.lower()
    if remove_unlinked or "dbp15k" in lowered or "dwy100k" in lowered:
        raise Unsupported("remove_unlinked / DBP15K / DWY100K layouts")
    if mode not in ("mapping", "sharing", "swapping"):
        mode = "mapping"                       # kgs.py: every mode other than 'sharing' uses mapping ids
    t0 = time.time()
    path = None
    if use_cache and os.environ.get("OEA_NO_DATASET_CACHE") != "1":
        path = os.path.join(cache_dir(), _signature(folder, division, mode, ordered) + ".npz")
        if os.path.exists(path):
            with np.load(path, allow_pickle=False) as z:
                parts = {k: z[k] for k in z.files}
            kgs = assemble(parts)
            if verbose:
                print("dataset arrays loaded from cache %s in %.2f s" % (path, time.time() - t0))
            return kgs
    parts = build(folder, division, mode, ordered)
    if path is not None:
        try:
            os.makedirs(os.path.dirname(path), exist_ok=True)
            tmp = path + ".%d.tmp.npz" % os.getpid()
            np.savez(tmp, **parts)
            os.replace(tmp, path)
        except OSError:
            pass                                # a read-only cache location only costs the next run its parse
    kgs = assemble(parts)
    if verbose:
        print("dataset parsed into arrays in %.2f s" % (time.time() - t0))
    return kgs
