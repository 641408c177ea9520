"""Device-side negative sampling (SURVEY 8f, next row 2): the reference's
getTrainTripleBatch / getNegRatings (utils/data.py:12-85) as two kernels over a device hash
set of the known triples / ratings.  The KG sampler emits the group-compact corrupt-id format
consumed by rank_loss_corrupt / loss_step_corrupt / SparseRowOptimizer.step_corrupt."""
import ctypes as C

import torch

from . import _lib
from . import functional as KF


class _KnownSet:
    def __init__(self, keys, device):
        lib = _lib.load()
        keys = keys.to(device=device, dtype=torch.int64).contiguous()
        self.capacity = int(lib.kgrec_hashset_capacity(keys.numel()))
        self.table = torch.empty(self.capacity, dtype=torch.int64, device=device)
        _lib.check(lib.kgrec_hashset_build(KF._ptr(keys), keys.numel(), KF._ptr(self.table), self.capacity, KF._stream()))
        KF.count_launches(1)


class _Checked:
    """status word shared by both samplers: 2 = some key had no valid negative at all (the reference's
    rejection loop would never have returned there, utils/data.py:23-56, 64-85)."""

    def _status(self):
        if getattr(self, "status", None) is None:
            self.status = torch.zeros(1, dtype=torch.int32, device=self.device)
        return self.status

    def check(self):
        """Raise if a sample() since the last check found a key without any valid negative (device sync)."""
        if getattr(self, "status", None) is not None and int(self.status.item()) != 0:
            self.status.zero_()
            raise RuntimeError("kgrec_b200: a negative sampler key has no valid negative (every candidate is the "
                               "positive or a known triple / rating)")


class TripleNegativeSampler(_Checked):
    """known_triples: [n, 3] (h, t, r) integer tensor of every triple negatives must avoid (the
    drivers pass train + valid + test dicts when -filter_wrong_corrupted, the default), or None."""

    def __init__(self, n_ent, n_rel, known_triples=None, device="cuda"):
        self.n_ent, self.n_rel, self.device = int(n_ent), int(n_rel), torch.device(device)
        self.known = None
        if known_triples is not None:
            k = torch.as_tensor(known_triples, dtype=torch.int64)
            keys = (k[:, 0] * self.n_rel + k[:, 2]) * self.n_ent + k[:, 1]
            self.known = _KnownSet(keys, self.device)

    def sample(self, pos, n_neg, seed=0, state=None):
        """pos = (h, t, r) device index tensors -> int32 [len(h) * n_neg] corrupt ids.
        state (kgrec_b200.train.StepState): draw with the running step's seed, state.sample_seed + state.step, read on
        the device (kgrec_sample_corrupt_dev); `seed` is then not used."""
        h, t, r = (KF.as_index(x, self.device) for x in pos)
        out = torch.empty(h.numel() * n_neg, dtype=torch.int32, device=self.device)
        tab = self.known
        lib = _lib.load()
        args = (KF._ptr(h), KF._ptr(t), KF._ptr(r), KF._idx_bytes(h, t, r), h.numel(), n_neg, self.n_ent, self.n_rel,
                KF._ptr(tab.table) if tab else None, tab.capacity if tab else 0)
        tail = (KF._ptr(out), KF._ptr(self._status()), KF._stream())
        if state is None:
            _lib.check(lib.kgrec_sample_corrupt(*args, int(seed) & 0xFFFFFFFFFFFFFFFF, *tail))
        else:
            _lib.check(lib.kgrec_sample_corrupt_dev(*args, state.ptr, *tail))
        KF.count_launches(1)
        return out


class RatingNegativeSampler(_Checked):
    """known_ratings: [n, 2] (u, i) pairs negatives must avoid (train + eval dicts), or None.

    One deliberate difference from getNegRatings (utils/data.py:64-85): the reference also refuses an item already
    drawn as a negative earlier in the SAME batch (`neg_set`, data.py:66,79-82 -- SURVEY appendix B: with more
    positives than items it never returns).  The device sampler draws every negative independently: a batch-wide
    set would serialise the batch, and for I >> B the two distributions differ by O(B / I)."""

    def __init__(self, n_item, known_ratings=None, device="cuda"):
        self.n_item, self.device = int(n_item), torch.device(device)
        self.known = None
        if known_ratings is not None:
            k = torch.as_tensor(known_ratings, dtype=torch.int64)
            self.known = _KnownSet(k[:, 0] * self.n_item + k[:, 1], self.device)

    def sample(self, u, pi, n_neg, seed=0, state=None):
        """state: as TripleNegativeSampler.sample (kgrec_sample_neg_items_dev)."""
        u, pi = KF.as_index(u, self.device), KF.as_index(pi, self.device)
        out = torch.empty(u.numel() * n_neg, dtype=torch.int32, device=self.device)
        tab = self.known
        lib = _lib.load()
        args = (KF._ptr(u), KF._ptr(pi), KF._idx_bytes(u, pi), u.numel(), n_neg, self.n_item,
                KF._ptr(tab.table) if tab else None, tab.capacity if tab else 0)
        tail = (KF._ptr(out), KF._ptr(self._status()), KF._stream())
        if state is None:
            _lib.check(lib.kgrec_sample_neg_items(*args, int(seed) & 0xFFFFFFFFFFFFFFFF, *tail))
        else:
            _lib.check(lib.kgrec_sample_neg_items_dev(*args, state.ptr, *tail))
        KF.count_launches(1)
        return out
