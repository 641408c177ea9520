"""GraphedTrainLoop (kgrec_b200/train.py): complete training steps replayed from CUDA graphs against the same steps run
eagerly -- through the same device-state (`_dev`) entry points, and through the host-scalar
SparseRowOptimizer.step_corrupt / step_pairs with the seeds derived the same way.  The batches and the negatives are
the same ids; the values agree to float rounding only, because the dense gradient accumulators, the row lists of the
row-factored rec step and clip_grad_norm's total norm are atomic sums whose order changes from run to run (two eager
runs of the same steps differ the same way).  CPU tests: symbols, struct layout, argument validation and the host's
mirror of DeviceTrainIterator's epoch rule."""
import ctypes as C
import random

import numpy as np
import pytest
import torch

FAKE = 0x7000_0000_1000


# ---- CPU ------------------------------------------------------------------------------------------------------------
NEW = ("kgrec_step_advance", "kgrec_batch_gather", "kgrec_rows_mark_dev", "kgrec_rows_sqnorm_dev", "kgrec_rows_update_dev",
       "kgrec_sample_corrupt_dev", "kgrec_sample_neg_items_dev", "kgrec_rank_loss_step_dev", "kgrec_rec_rows_step_dev")


def test_step_state_symbols_are_exported():
    from kgrec_b200 import _lib
    lib = _lib.load()
    for name in NEW:
        assert name in _lib.EXPORTS and hasattr(lib, name)


def test_step_state_layout_matches_header():
    from kgrec_b200 import _lib
    S = _lib.StepState
    # int64 step, uint64 gumbel_seed, uint64 sample_seed, int32 epoch, float lr
    assert C.sizeof(S) == 32
    assert (S.step.offset, S.gumbel_seed.offset, S.sample_seed.offset, S.epoch.offset, S.lr.offset) == (0, 8, 16, 24, 28)


def test_c_abi_step_state_argument_validation_without_a_gpu():
    from kgrec_b200 import _lib
    lib = _lib.load()

    def err():
        return lib.kgrec_last_error().decode()
    assert lib.kgrec_step_advance(None, None, 1, None) != 0 and "NULL state" in err()
    assert lib.kgrec_step_advance(FAKE, None, -1, None) != 0
    cols = (C.c_void_p * 3)(FAKE, FAKE, FAKE)

    def gather(order=FAKE, n_order=100, cursor=FAKE, n_cols=3, idx_bytes=4, n_rows=100, batch=10):
        return lib.kgrec_batch_gather(order, n_order, cursor, cols, cols, n_cols, idx_bytes, n_rows, batch, None, None)
    for bad in (dict(order=None), dict(cursor=None), dict(n_cols=0), dict(n_cols=5), dict(idx_bytes=2), dict(n_rows=0),
                dict(batch=-1), dict(n_order=0)):
        assert gather(**bad) != 0 and "kgrec_batch_gather" in err(), bad
    assert gather(batch=0) == 0               # nothing to gather: no launch
    seg = _lib.MarkSeg(ids=FAKE, n=4, idx_bytes=4, marks=FAKE, rows=10)
    assert lib.kgrec_rows_mark_dev((_lib.MarkSeg * 1)(seg), 1, None, None, None) != 0 and "state is NULL" in err()
    assert lib.kgrec_rows_mark_dev((_lib.MarkSeg * 1)(seg), 9, FAKE, None, None) != 0 and "id segments" in err()
    tab = (_lib.OptTable * 1)(_lib.OptTable(table=FAKE, acc=FAKE, rows=10, dim=4))
    assert lib.kgrec_rows_sqnorm_dev(tab, 1, None, FAKE, None) != 0 and "state is NULL" in err()
    assert lib.kgrec_rows_sqnorm_dev(tab, 1, FAKE, None, None) != 0 and "sqnorm is NULL" in err()
    assert lib.kgrec_rows_update_dev(tab, 1, None, 0, 1e-8, 0.9, 0.999, 0.0, None, 0.0, None) != 0 and "state is NULL" in err()
    assert lib.kgrec_rows_update_dev(tab, 1, FAKE, 2, 1e-8, 0.9, 0.999, 0.0, None, 0.0, None) != 0 and "state missing" in err()
    assert lib.kgrec_rows_update_dev(tab, 9, FAKE, 0, 1e-8, 0.9, 0.999, 0.0, None, 0.0, None) != 0 and "tables per call" in err()
    assert lib.kgrec_sample_corrupt_dev(FAKE, FAKE, FAKE, 4, 8, 1, 100, 5, None, 0, None, FAKE, None, None) != 0
    assert "state is NULL" in err()
    assert lib.kgrec_sample_corrupt_dev(FAKE, FAKE, FAKE, 4, 8, 0, 100, 5, None, 0, FAKE, FAKE, None, None) != 0
    assert "bad arguments" in err()
    assert lib.kgrec_sample_neg_items_dev(FAKE, FAKE, 4, 8, 1, 100, None, 0, None, FAKE, None, None) != 0
    assert "state is NULL" in err()
    assert lib.kgrec_sample_neg_items_dev(FAKE, FAKE, 3, 8, 1, 100, None, 0, FAKE, FAKE, None, None) != 0
    t = _lib.Tables(dim=64, ld=64, n_user=50, n_item=40, n_pref=4, user=FAKE, item=FAKE, pref=FAKE, pref_norm=FAKE)
    g = _lib.Grads(mode=1, user=FAKE, item=FAKE, pref=FAKE, pref_norm=FAKE)
    assert lib.kgrec_rank_loss_step_dev(C.byref(t), _lib.TUP, FAKE, FAKE, None, FAKE, FAKE, None, 4, 8, 1, 8, _lib.LOSS_BPR,
                                        -1.0, 1.0, None, None, FAKE, FAKE, FAKE, C.byref(g), None, None, None, FAKE, None,
                                        None) != 0 and "state is NULL" in err()
    assert lib.kgrec_rank_loss_step_dev(C.byref(t), 99, FAKE, FAKE, None, FAKE, FAKE, None, 4, 8, 1, 8, _lib.LOSS_BPR,
                                        -1.0, 1.0, None, FAKE, FAKE, FAKE, FAKE, C.byref(g), None, None, None, FAKE, None,
                                        None) != 0 and "unknown model" in err()

    def rows(state=FAKE, model=_lib.TUP, n_neg=1):
        return lib.kgrec_rec_rows_step_dev(C.byref(t), model, FAKE, FAKE, FAKE, 4, 8, n_neg, 8, _lib.LOSS_BPR, -1.0, 1.0,
                                           FAKE, FAKE, state, FAKE, 0, C.byref(g), FAKE, FAKE, FAKE, FAKE, None, None,
                                           None, None)
    assert rows(state=None) != 0 and "state is NULL" in err()
    assert rows(model=_lib.TRANSE) != 0 and "TUP / KTUP" in err()
    assert rows(n_neg=40) != 0 and "1..31 negatives" in err()


@pytest.mark.parametrize("seed", range(6))
def test_replay_plan_mirrors_the_iterator_epoch_rule(seed):
    """The schedule GraphedTrainLoop.run follows, against DeviceTrainIterator itself (on the CPU): the batch every step
    draws, and the iterators' positions afterwards."""
    from kgrec_b200.data import DeviceTrainIterator
    from kgrec_b200.train import replay_plan
    rnd = random.Random(seed)
    for _ in range(20):
        ktup = rnd.random() < 0.4
        names = ("rec", "kg") if ktup else ("kg",)
        its, twins = {}, {}
        for k in names:
            n, bs, rep = rnd.randint(1, 60), rnd.randint(1, 12), rnd.randint(1, 3)
            bs = min(bs, n)
            data = torch.arange(n).view(-1, 1)
            its[k] = DeviceTrainIterator(data, bs, negtive_samples=rep, device="cpu", seed=seed)
            twins[k] = DeviceTrainIterator(data, bs, negtive_samples=rep, device="cpu", seed=seed)
        S = rnd.choice([0, 1, 2, 3, 7, 10, 13]) if not ktup else rnd.choice([0, 1, 10, 20])
        ratio = rnd.choice([0.3, 0.5, 0.7])
        kinds = (lambda g: "rec" if g % 10 < 10 * ratio else "kg") if ktup else (lambda g: "kg")
        n_steps = rnd.randint(1, 80)
        plan = replay_plan(kinds, {k: it.start for k, it in its.items()}, {k: it.n for k, it in its.items()},
                           {k: it.batch_size for k, it in its.items()}, n_steps, S)
        assert sum(s for _, s in plan) == n_steps
        assert all(s in (1, S) for _, s in plan)
        g = 0
        for reshuffle, steps in plan:
            for k in reshuffle:           # what _Source.new_epoch does
                it = its[k]
                it.start, it.epoch = -it.batch_size, it.epoch + 1
                it._shuffle()
            for i in range(steps):
                it, twin = its[kinds(g + i)], twins[kinds(g + i)]
                want = next(twin)[0]
                it.start += it.batch_size
                got = it.cols[0][it.order[it.start:it.start + it.batch_size]]
                assert torch.equal(got, want)
                # `it` only starts epochs between replays: the eager iterator never starts one inside a replay
                assert twin.epoch == it.epoch
            g += steps
        for k in names:
            assert (its[k].start, its[k].epoch) == (twins[k].start, twins[k].epoch)


# ---- GPU ------------------------------------------------------------------------------------------------------------
D = 64
N_ENT, N_REL, N_TRIPLES = 700, 11, 2600
N_USER, N_ITEM, N_PREF, N_RATINGS = 300, 200, 6, 2600
BATCH, N_STEPS = 256, 25          # 10 batches an epoch: 2.5 epochs


def _kg_data(rng, n_ent=N_ENT, bad=False):
    t = np.stack([rng.randint(0, n_ent, N_TRIPLES), rng.randint(0, n_ent, N_TRIPLES), rng.randint(0, N_REL, N_TRIPLES)], 1)
    if bad:
        t[::50, 1] = n_ent + 5
    return t


def _rec_data(rng):
    return np.stack([rng.randint(0, N_USER, N_RATINGS), rng.randint(0, N_ITEM, N_RATINGS)], 1)


def _setup(case, opt_type="Adagrad", seed=0, bad=False):
    import kgrec_b200 as K
    from kgrec_b200.data import DeviceTrainIterator
    from kgrec_b200.optim import SparseRowOptimizer
    from kgrec_b200.sampling import RatingNegativeSampler, TripleNegativeSampler
    model_name, l1, gumbel = case["model"], case.get("l1", False), case.get("gumbel", False)
    rng = np.random.RandomState(seed)
    torch.manual_seed(seed)
    out = {"n_neg": case.get("n_neg", 1)}
    if model_name in ("transe", "transh", "transr"):
        cls = {"transe": K.TransEModel, "transh": K.TransHModel, "transr": K.TransRModel}[model_name]
        model = cls(l1, D, N_ENT, N_REL)
        triples = _kg_data(rng, bad=bad)
        out["it"] = DeviceTrainIterator(triples, BATCH, device="cuda", seed=seed + 1)
        out["sampler"] = TripleNegativeSampler(N_ENT, N_REL, known_triples=None if bad else triples)
    elif model_name == "tup":
        model = K.TransUPModel(l1, D, N_USER, N_ITEM, N_PREF, gumbel)
        ratings = _rec_data(rng)
        out["it"] = DeviceTrainIterator(ratings, BATCH, device="cuda", seed=seed + 1)
        out["sampler"] = RatingNegativeSampler(N_ITEM, known_ratings=ratings)
    else:
        n_ent = 400
        ents = rng.permutation(n_ent)[:N_ITEM]
        new_map = {i: (int(ents[i]) if i % 10 < 7 else -1, i) for i in range(N_ITEM)}
        model = K.jTransUPModel(l1, D, N_USER, N_ITEM, n_ent, N_PREF, {i: i for i in range(N_ITEM)}, new_map, False, gumbel)
        ratings, triples = _rec_data(rng), _kg_data(rng, n_ent=n_ent)
        triples[:, 2] %= N_PREF
        out["it"] = DeviceTrainIterator(ratings, BATCH, device="cuda", seed=seed + 1)
        out["sampler"] = RatingNegativeSampler(N_ITEM, known_ratings=ratings)
        out["kg_it"] = DeviceTrainIterator(triples, 200, device="cuda", seed=seed + 2)      # 13 batches an epoch
        out["kg_sampler"] = TripleNegativeSampler(n_ent, N_PREF, known_triples=triples)
    out["model"] = model
    out["opt"] = SparseRowOptimizer(model, optimizer_type=opt_type, lr=0.01 if opt_type != "SGD" else 0.05,
                                    l2_lambda=1e-3, clip=1.0)
    return out


def _loop(env, case, S):
    from kgrec_b200.train import GraphedTrainLoop
    kw = dict(steps_per_graph=S, reg=case.get("reg", False), sample_seed=77)
    if "kg_it" in env:
        kw.update(kg_iterator=env["kg_it"], kg_sampler=env["kg_sampler"], joint_ratio=case["ratio"], kg_lambda=0.5)
    return GraphedTrainLoop(env["model"], env["opt"], env["it"], env["sampler"], env["n_neg"], **kw)


def _host_steps(env, case, n_steps, step0=0):
    """The same steps through the host-scalar methods: seeds sample_seed + t and the model's own Gumbel sequence."""
    opt, model = env["opt"], env["model"]
    ktup = "kg_it" in env
    losses = []
    for g in range(step0, step0 + n_steps):
        rec = ktup and g % 10 < 10 * case["ratio"] or case["model"] == "tup"
        s = opt.t + 1
        if rec:
            u, i = next(env["it"])
            ni = env["sampler"].sample(u, i, env["n_neg"], seed=77 + s)
            out, _ = opt.step_pairs((u, i), (u, ni), target=-1.0, reg=case.get("reg", False))
        else:
            it, smp = (env["kg_it"], env["kg_sampler"]) if ktup else (env["it"], env["sampler"])
            pos = next(it)
            corrupt = smp.sample(pos, env["n_neg"], seed=77 + s)
            out = opt.step_corrupt(pos, corrupt, margin=1.0, reg=case.get("reg", False), grad_loss=0.5 if ktup else 1.0)
        losses.append(out.view(-1)[:1])
    return torch.cat(losses)


def _snapshot(env):
    opt = env["opt"]
    snap = {"w." + k: v.detach().clone() for k, v in env["model"].named_parameters()}
    for name, d in (("acc", opt.acc), ("s1", opt.s1), ("s2", opt.s2)):
        snap.update({name + "." + k: v.clone() for k, v in d.items() if v is not None})
    return snap


def _assert_same(a, b, tol=2e-5):
    """Equal up to the reordering of atomic float sums over 25 steps (a wrong seed, batch, epoch, lr or step count moves
    the tables by orders of magnitude more)."""
    assert a.keys() == b.keys()
    for k in a:
        torch.testing.assert_close(a[k], b[k], rtol=tol, atol=tol, msg=lambda m: "%s: %s" % (k, m))


CASES = {
    "transe_l1": dict(model="transe", l1=True, n_neg=3),
    "transe_l2": dict(model="transe", l1=False, n_neg=3),
    "transh_reg": dict(model="transh", l1=True, reg=True),
    "transr": dict(model="transr", l1=False),
    "tup_soft_rows": dict(model="tup", rows="force"),
    "tup_soft_pairs": dict(model="tup", rows="0"),
    "tup_gumbel_rows": dict(model="tup", gumbel=True, rows="force"),
    "tup_gumbel_pairs": dict(model="tup", gumbel=True, rows="0"),
    "ktup_0.5": dict(model="ktup", ratio=0.5, reg=True, rows="0"),
    "ktup_0.3_rows": dict(model="ktup", ratio=0.3, reg=True, rows="force"),
}


def _graphed_eager_host(monkeypatch, case, opt_type, S, n_steps=N_STEPS):
    if "rows" in case:
        monkeypatch.setenv("KGREC_REC_ROWS", case["rows"])
    results = []
    for mode in (S, 0, "host"):
        env = _setup(case, opt_type)
        if mode == "host":
            loss = _host_steps(env, case, n_steps)
        else:
            loss = _loop(env, case, mode).run(n_steps)
        torch.cuda.synchronize()
        snap = _snapshot(env)
        snap["loss"] = loss
        results.append((snap, env))
    return results


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_graphed_loop_matches_eager(monkeypatch, name):
    case = CASES[name]
    S = 10 if case["model"] == "ktup" else 7          # 7 does not divide the 10-batch epoch
    (g, genv), (e, eenv), (h, henv) = _graphed_eager_host(monkeypatch, case, "Adagrad", S)
    _assert_same(g, e)
    _assert_same(g, h)
    for k in ("it", "kg_it"):
        if k in genv:
            assert (genv[k].start, genv[k].epoch) == (henv[k].start, henv[k].epoch)
    assert genv["opt"].t == henv["opt"].t == N_STEPS
    genv["sampler"].check()
    genv["model"].check_indices()


@pytest.mark.gpu
@pytest.mark.parametrize("opt_type", ["SGD", "Adagrad", "Adam"])
def test_graphed_loop_optimizers(monkeypatch, opt_type):
    (g, _), (e, _), (h, _) = _graphed_eager_host(monkeypatch, CASES["transe_l2"], opt_type, 4)
    _assert_same(g, e)
    _assert_same(g, h)


@pytest.mark.gpu
def test_set_lr_takes_effect_on_the_next_step():
    case = CASES["transh_reg"]
    a, b = _setup(case), _setup(case)
    la = _loop(a, case, 7)
    la.run(9)
    la.set_lr(0.002)
    la.run(12)
    b_loss = _host_steps(b, case, 9)
    b["opt"].lr = 0.002
    b_loss = _host_steps(b, case, 12, step0=9)
    torch.cuda.synchronize()
    _assert_same(_snapshot(a), _snapshot(b))
    assert la.state.read()["lr"] == pytest.approx(0.002)
    assert la.state.read()["step"] == 21


@pytest.mark.gpu
def test_out_of_range_id_raises_through_check():
    case = CASES["transe_l1"]
    env = _setup(case, bad=True)
    loop = _loop(env, case, 7)
    loop.run(N_STEPS)
    with pytest.raises(IndexError):
        loop.check()
    loop.check()                    # the status word is cleared by the check that raised
    assert torch.isfinite(env["model"].ent_embeddings.weight).all()
