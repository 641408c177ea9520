"""On-disk formats around the hot path (SURVEY 8f, next row 4).

The reference re-parses its TSV files into Python lists and dicts of sets on every start
(jTransUP/data/load_triple_data.py:5-30, load_rating_data.py:19-38) and feeds the kernels from
those.  Here the same files are parsed once into int32 arrays, cached as one `.npz` next to the
TSV, and exposed in the forms the CUDA path consumes: packed 64-bit keys for the device hash
set (sampling.py), CSR filter lists for the top-K kernel (evaluation.build_filter_csr works on
the dict view, also provided), and the reference's own dict / list views for unchanged code.
Checkpoints use the reference's layout (utils/trainer.py:109-142) so they interchange.
"""
import os

import numpy as np
import torch


def _parse_int_tsv(path, n_cols):
    rows = []
    with open(path, "r", encoding="utf-8") as fin:
        for line in fin:
            parts = line.strip().split("\t")
            if len(parts) != n_cols:          # the reference skips malformed lines the same way
                continue
            rows.append([int(x) for x in parts])
    return np.asarray(rows, dtype=np.int32).reshape(-1, n_cols)


def _cached(path, n_cols, use_cache):
    cache = path + ".kgrec.npz"
    if use_cache and os.path.exists(cache) and os.path.getmtime(cache) >= os.path.getmtime(path):
        with np.load(cache) as z:
            return z["rows"]
    rows = _parse_int_tsv(path, n_cols)
    if use_cache:
        try:
            np.savez(cache, rows=rows)
        except OSError:
            pass                                   # read-only dataset directory: parse every time
    return rows


class TripleFile:
    """`train.dat` / `valid.dat` / `test.dat` of a KG: lines `head \\t tail \\t relation`
    (README.md:45-55; load_triple_data.py:5-30)."""

    def __init__(self, path, use_cache=True):
        self.rows = _cached(path, 3, use_cache)    # [n, 3] int32: h, t, r

    @property
    def total(self):
        return len(self.rows)

    def as_list(self):
        return [tuple(int(v) for v in r) for r in self.rows]

    def head_dict(self):
        """{(t, r): set(heads)} as loadTriples builds it."""
        out = {}
        for h, t, r in self.rows.tolist():
            out.setdefault((t, r), set()).add(h)
        return out

    def tail_dict(self):
        out = {}
        for h, t, r in self.rows.tolist():
            out.setdefault((h, r), set()).add(t)
        return out

    def tensor(self, device="cpu"):
        return torch.from_numpy(self.rows.astype(np.int64)).to(device)


class RatingFile:
    """`train.dat` / eval files of the recommendation task: `user \\t item \\t rating`
    (load_rating_data.py:19-38; the rating value is read and dropped, as in the reference)."""

    def __init__(self, path, use_cache=True):
        self.rows = _cached(path, 3, use_cache)[:, :2].copy()   # [n, 2] int32: u, i

    @property
    def total(self):
        return len(self.rows)

    def as_list(self):
        return [tuple(int(v) for v in r) for r in self.rows]

    def rating_dict(self):
        out = {}
        for u, i in self.rows.tolist():
            out.setdefault(u, set()).add(i)
        return out

    def tensor(self, device="cpu"):
        return torch.from_numpy(self.rows.astype(np.int64)).to(device)


def csr_from_dicts(keys, dicts, device="cpu", id_lo=0, id_hi=None):
    """Vectorised form of evaluation.build_filter_csr for large eval sets."""
    ptr = np.zeros(len(keys) + 1, dtype=np.int64)
    chunks = []
    for n, key in enumerate(keys):
        s = set()
        for d in dicts or ():
            if key in d:
                s.update(d[key])
        row = np.fromiter((i for i in s if i >= id_lo and (id_hi is None or i < id_hi)), dtype=np.int32)
        row.sort()
        chunks.append(row)
        ptr[n + 1] = ptr[n] + len(row)
    ids = np.concatenate(chunks) if chunks and ptr[-1] else np.zeros(1, dtype=np.int32)
    return torch.from_numpy(ptr).to(device), torch.from_numpy(ids).to(device)


# ---- relation categories of link prediction (1-1 / 1-N / N-1 / N-N) ------------------------------------------
REL_CATEGORIES = ("1-1", "1-N", "N-1", "N-N")
_REL_TYPE_LABELS = {"one2one": 0, "one2many": 1, "many2one": 2, "many2many": 3}


def relation_categories(triples, n_rel):
    """int8 [n_rel]: the category of every relation, 0 = 1-1, 1 = 1-N, 2 = N-1, 3 = N-N, -1 = absent from `triples`.

    splitRelationType (preprocessTriples.py:14-56) restated on an [n, 3] (h, t, r) array; the reference passes
    train + valid + test (preprocessTriples.py:253).  avg_head = round(mean over the (t, r) keys of r of |heads|),
    avg_tail likewise over the (h, r) keys, with Python 3's round (half to even, as np.rint); a relation is N-N when
    both are > 1, N-1 when only avg_head is, 1-N when only avg_tail is, 1-1 otherwise."""
    a = np.asarray(triples, dtype=np.int64).reshape(-1, 3)
    out = np.full(n_rel, -1, dtype=np.int8)
    if not a.size:
        return out
    if a[:, 2].min() < 0 or a[:, 2].max() >= n_rel:
        raise IndexError("kgrec_b200: a relation id of the triples is outside [0, n_rel)")
    trip = np.unique(a, axis=0)                        # |heads| of (t, r) counts distinct h, as the reference's sets do

    def avg(key_a, key_b):
        keys, n_per_key = np.unique(np.stack([key_a, key_b], 1), axis=0, return_counts=True)
        rel = keys[:, 1]
        s = np.bincount(rel, weights=n_per_key, minlength=n_rel)
        k = np.bincount(rel, minlength=n_rel)
        return np.rint(s / np.maximum(k, 1)), k > 0
    h, t, r = trip[:, 0], trip[:, 1], trip[:, 2]
    avg_head, present = avg(t, r)
    avg_tail, _ = avg(h, r)
    many_h, many_t = avg_head > 1, avg_tail > 1
    cat = np.where(many_h, np.where(many_t, 3, 2), np.where(many_t, 1, 0))
    out[present] = cat[present]
    return out


def load_relation_types(path, n_rel=None):
    """The reference's `relation_type.dat` (lines `one2one|one2many|many2one|many2many \\t r \\t r ...`, written by
    preprocessTriples.py:280-284) as the int8 array relation_categories returns, read by each line's label.  n_rel
    defaults to 1 + the largest relation id in the file.  (The reference's own loadRelationType assigns lines by
    their position among the non-empty ones, so an empty category shifts the later ones: SURVEY appendix B.)"""
    rel = {}
    with open(path, "r", encoding="utf-8") as fin:
        for line in fin:
            parts = line.strip().split("\t")
            if not parts[0]:
                continue
            if parts[0] not in _REL_TYPE_LABELS:
                raise ValueError("kgrec_b200: unknown relation type label %r in %s" % (parts[0], path))
            for x in parts[1:]:
                rel[int(x)] = _REL_TYPE_LABELS[parts[0]]
    n = n_rel if n_rel is not None else 1 + max(rel, default=-1)
    out = np.full(n, -1, dtype=np.int8)
    for r, c in rel.items():
        out[r] = c
    return out


def save_checkpoint(path, model, optimizer=None, step=0, best_step=0, best_dev_performance=0.0):
    """The reference's checkpoint dict (utils/trainer.py:115-122), tensors on the CPU."""
    sd = {k: v.detach().cpu() for k, v in model.state_dict().items()}
    torch.save({"step": step, "best_step": best_step, "best_dev_performance": best_dev_performance,
                "model_state_dict": sd,
                "optimizer_state_dict": optimizer.state_dict() if optimizer is not None else {}}, path)


def load_checkpoint(path, model, optimizer=None, trusted=True):
    """ModelTrainer.load (utils/trainer.py:128-142): strict=False state_dict load; returns the
    bookkeeping fields.  Works on checkpoints written by the reference trainer as well: those carry
    `best_dev_performance` as a numpy scalar (trainer.py:115-122 saves what np.mean returned), which
    torch >= 2.6's default weights-only unpickler refuses -- the reference's own trainer unpickles the
    file in full, and so does this function for a `trusted` (local, self-written) file after the safe
    attempt fails.  trusted=False keeps the weights-only behaviour and raises on such files."""
    import pickle
    try:
        ck = torch.load(path, map_location="cpu", weights_only=True)
    except pickle.UnpicklingError:
        if not trusted:
            raise
        ck = torch.load(path, map_location="cpu", weights_only=False)
    model.load_state_dict(ck["model_state_dict"], strict=False)
    if optimizer is not None and ck.get("optimizer_state_dict"):
        optimizer.load_state_dict(ck["optimizer_state_dict"])
    return ck.get("step", 0), ck.get("best_step", 0), ck.get("best_dev_performance", 0.0)


# ---- vocabularies and the item <-> entity alignment of the joint models -------------------------------------
def load_vocab(path):
    """`u_map.dat` / `i_map.dat` / `e_map.dat` / `r_map.dat`: lines `mapped_id \\t original_id`;
    returns {original_id (str): mapped_id (int)} as loadVocab does (load_rating_data.py:6-16,
    load_triple_data.py:32-43); lines without exactly two fields are skipped."""
    vocab = {}
    with open(path, "r", encoding="utf-8") as fin:
        for line in fin:
            parts = line.strip().split("\t")
            if len(parts) != 2:
                continue
            vocab[parts[1]] = int(parts[0])
    return vocab


def load_item_kg_map(path):
    """`i2kg_map.tsv`: lines `original item id \\t title \\t entity uri` -> (i2kg, kg2i) as loadR2KgMap
    (load_kg_rating_data.py:5-18)."""
    i2kg, kg2i = {}, {}
    with open(path, "r", encoding="utf-8") as fin:
        for line in fin:
            parts = line.strip().split("\t")
            if len(parts) != 3:
                continue
            i2kg[parts[0]] = parts[2]
            kg2i[parts[2]] = parts[0]
    return i2kg, kg2i


def rebuild_entity_item_vocab(map1, map2, links):
    """rebuildEntityItemVocab (load_kg_rating_data.py:21-48): the joint vocabulary of entities (map1: uri -> id)
    and items (map2: original id -> id) linked by `links` (uri -> original item id).  Returns
    (new_map {joint index: (entity id | -1, item id | -1)}, remap1 {entity id: joint index},
    remap2 {item id: joint index}, number of aligned pairs) -- the reference's return values, built with the
    same iteration order (dict order of map1, then of map2)."""
    new_map, remap1, remap2, has_map2 = {}, {}, {}, {}
    index = 0
    for org1, id1 in map1.items():
        mapped2 = -1
        org2 = links.get(org1)
        if org2 is not None and org2 in map2:
            mapped2 = map2[org2]
            has_map2[org2] = index
        new_map[index] = (id1, mapped2)
        remap1[id1] = index
        index += 1
    for org2, id2 in map2.items():
        if org2 in has_map2:
            remap2[id2] = has_map2[org2]
            continue
        new_map[index] = (-1, id2)
        remap2[id2] = index
        index += 1
    return new_map, remap1, remap2, len(has_map2)


def item_to_entity_table(item_total, pad, i_remap, ikg_map):
    """The device lookup jTransUPModel needs (item -> aligned entity row, unaligned -> the padding row):
    paddingItems (jTransUP.py:114-120) over every item, vectorised (models/jTransUP.build_item2ent)."""
    from .models.jTransUP import build_item2ent
    return build_item2ent(item_total, pad, i_remap, ikg_map)


class JointDataset:
    """Everything `load_kg_rating_data.load_data` (load_kg_rating_data.py:51-65) returns, parsed once:
    rating / triple files as int32 arrays (with the reference's list / dict views on demand), the four
    vocabularies, and the item <-> entity alignment."""

    def __init__(self, data_path, rec_eval_files=(), kg_eval_files=(), use_cache=True):
        kg = os.path.join(data_path, "kg")
        self.rating_train = RatingFile(os.path.join(data_path, "train.dat"), use_cache)
        self.rating_eval = [RatingFile(os.path.join(data_path, f), use_cache) for f in rec_eval_files]
        self.triple_train = TripleFile(os.path.join(kg, "train.dat"), use_cache)
        self.triple_eval = [TripleFile(os.path.join(kg, f), use_cache) for f in kg_eval_files]
        self.u_map = load_vocab(os.path.join(data_path, "u_map.dat"))
        self.i_map = load_vocab(os.path.join(data_path, "i_map.dat"))
        self.e_map = load_vocab(os.path.join(kg, "e_map.dat"))
        self.r_map = load_vocab(os.path.join(kg, "r_map.dat"))
        self.i2kg, self.kg2i = load_item_kg_map(os.path.join(data_path, "i2kg_map.tsv"))
        self.ikg_map, self.e_remap, self.i_remap, self.aligned = rebuild_entity_item_vocab(self.e_map, self.i_map, self.kg2i)

    def totals(self):
        """(user_total, item_total, entity_total, relation_total) as knowledgable_recommendation.run computes
        them for -noshare_embeddings (knowledgable_recommendation.py:455-458)."""
        return (max(len(self.u_map), max(self.u_map.values())), max(len(self.i_remap), max(self.i_remap.keys())),
                max(len(self.e_remap), max(self.e_remap.keys())), max(len(self.r_map), max(self.r_map.values())))
