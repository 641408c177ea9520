"""TransR's step kernels with the KG drivers' regularisers fused in (kgrec_corrupt_loss_step, reg_flags = 1).

knowledge_representation.py:189-204 trains every KG model on marginLoss plus normLoss over the entity rows of
cat[ph, pt, nh, nt] and the relation rows of cat[pr, nr].  For TransR the norms are those of the RAW ent / rel rows
(the reference regularises model.ent_embeddings / rel_embeddings, not the projections) and proj has no term.

The reference side here is a float64 torch-autograd restatement of that loss on a dense copy of the tables: the TransR
score (transR.py:65-78, misc.py:21-26), marginLoss and normLoss (loss.py:8-23), per batch of batch_pos positives with
nh / nt / nr expanded from the corrupted ids.  Rows are scaled to 1.05 / 0.95 (alternating), so every row is off the
kink of max(|x|^2 - 1, 0).
CPU tests: the entry point's host-side checks of reg_flags for TransR."""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

FAKE = 0x7000_0000_1000
ERR_INVALID, ERR_UNSUPPORTED = 1, 2          # KGREC_ERR_* (include/kgrec_b200.h)


# ---- CPU ------------------------------------------------------------------------------------------------------------
def test_c_abi_transr_reg_flags_without_a_gpu():
    from kgrec_b200 import _lib
    lib = _lib.load()

    def err():
        return lib.kgrec_last_error().decode()
    t = _lib.Tables(dim=100, ld=100, n_ent=50, n_rel=7, ent=FAKE, rel=FAKE, proj=FAKE)
    g = _lib.Grads(mode=1, ent=FAKE, rel=FAKE, proj=FAKE)

    def step(n_pos=4, n_neg=2, loss=_lib.LOSS_MARGIN, reg=1):
        return lib.kgrec_corrupt_loss_step(C.byref(t), _lib.TRANSR, FAKE, FAKE, FAKE, 4, n_pos, FAKE, n_neg, 4, loss, 1.0, 1.0,
                                           reg, FAKE, FAKE, FAKE, C.byref(g), None, None, FAKE, None, None)
    assert step(n_pos=0) == 0                                                   # accepted: nothing to launch
    assert step(reg=2) == ERR_INVALID and "reg_flags must be 0 or 1" in err()
    assert step(loss=_lib.LOSS_BPR) == ERR_UNSUPPORTED and "margin loss" in err()
    assert step(n_neg=15) == ERR_UNSUPPORTED and "at most 14 negatives" in err()


# ---- GPU: the float64 restatement of the driver's loss ---------------------------------------------------------------
def _ids(h, t, r, corrupt, K):
    c = corrupt.long()
    head = c < 0
    cid = torch.where(head, ~c, c)
    nh = torch.where(head, cid, h.long().repeat_interleave(K))
    nt = torch.where(head, t.long().repeat_interleave(K), cid)
    return h.long(), t.long(), r.long(), nh, nt, r.long().repeat_interleave(K)


def _residuals(ent, rel, proj, h, t, r):
    """M_r h + r - M_r t per triple (projection_transR_pytorch: M = proj[r].view(d, d) times the column h), one
    relation at a time, in the triples' order."""
    d = ent.shape[1]
    parts, where = [], []
    for rid in torch.unique(r).tolist():
        sel = (r == rid).nonzero().view(-1)
        M = proj[rid].view(d, d)
        parts.append(ent[h[sel]] @ M.t() + rel[rid] - ent[t[sel]] @ M.t())
        where.append(sel)
    return torch.cat(parts)[torch.argsort(torch.cat(where))]


def _score(ent, rel, proj, h, t, r, l1):
    e = _residuals(ent, rel, proj, h, t, r)
    return e.abs().sum(1) if l1 else (e ** 2).sum(1)


def _norm_loss(x):
    return torch.clamp((x ** 2).sum(1) - 1.0, min=0).sum()


def ref_step(w, pos, corrupt, K, bp, margin, l1, grad_loss):
    """Per-batch losses, scores and the float64 gradients of grad_loss * sum(losses) (knowledge_representation.py:189-204)."""
    ent, rel, proj = (w[k].detach().double().cpu().requires_grad_() for k in ("ent", "rel", "proj"))
    h, t, r, nh, nt, nr = (x.cpu() for x in _ids(*pos, corrupt, K))
    sp = _score(ent, rel, proj, h, t, r, l1)
    sn = _score(ent, rel, proj, nh, nt, nr, l1)
    n_pos = h.numel()
    losses = []
    for b in range((n_pos + bp - 1) // bp):
        ps, ns = slice(b * bp, (b + 1) * bp), slice(b * bp * K, (b + 1) * bp * K)
        lm = torch.clamp(sp[ps].repeat_interleave(K) - sn[ns] + margin, min=0).sum()
        reg = _norm_loss(ent[torch.cat([h[ps], t[ps], nh[ns], nt[ns]])]) + _norm_loss(rel[torch.cat([r[ps], nr[ns]])])
        losses.append(lm + reg)
    losses = torch.stack(losses)
    (grad_loss * losses.sum()).backward()
    # L1 residual components within float32 rounding of 0 may take either sign on the two sides
    with torch.no_grad():
        n_amb = int((_residuals(ent, rel, proj, h, t, r).abs() < 1e-6).sum() +
                    (_residuals(ent, rel, proj, nh, nt, nr).abs() < 1e-6).sum()) if l1 else 0
    return dict(loss=losses.detach(), pos=sp.detach(), neg=sn.detach(), ent=ent.grad, rel=rel.grad, proj=proj.grad, n_amb=n_amb)


def _dense(g):
    return (g.to_dense() if g.is_sparse else g).detach().double().cpu()


def _close(got, want, what, rtol=2e-3, atol_rel=2e-4, max_outliers=0):
    got, want = got.double().cpu(), want.double().cpu()
    atol = atol_rel * max(1.0, float(want.abs().max()))
    bad = int(((got - want).abs() > atol + rtol * want.abs()).sum())
    assert bad <= max_outliers, "%s: %d elements off (max |diff| %.3g, atol %.3g)" % (what, bad, float((got - want).abs().max()), atol)


def _make(d, E, R, l1, seed, scale=None):
    import kgrec_b200 as K
    torch.manual_seed(seed)
    m = K.TransRModel(l1, d, E, R)
    with torch.no_grad():
        for tab, n in ((m.ent_embeddings.weight, E), (m.rel_embeddings.weight, R)):
            s = torch.where(torch.arange(n, device=tab.device) % 2 == 0, 1.05, 0.95) if scale is None else \
                torch.full((n,), scale, device=tab.device)
            tab.mul_(s.view(-1, 1) / tab.norm(dim=1, keepdim=True))
    return m


def _inputs(E, R, n_pos, K, seed, idx, repeats=True):
    rng = np.random.RandomState(seed)
    h, t, r = rng.randint(0, E, n_pos), rng.randint(0, E, n_pos), rng.randint(0, R, n_pos)
    ce = rng.randint(0, E, n_pos * K)
    if repeats:                  # the same entity several times in one group and one batch
        h[1], t[2], t[0] = h[0], h[0], h[0]
        ce[0], ce[min(1, K * n_pos - 1)] = h[0], t[3]
        r[1] = r[0]
    head = rng.rand(n_pos * K) < 0.4
    dt = torch.int64 if idx == "int64" else torch.int32
    pos = tuple(torch.as_tensor(x, dtype=dt, device="cuda") for x in (h, t, r))
    return pos, torch.as_tensor(np.where(head, ~ce, ce).astype(np.int32), device="cuda")


def _kernels_that_ran(fn):
    """Names of the CUDA events fn() leaves in a profile.  Now and then the profiler loses a capture's kernel records
    (only runtime calls and an "Activity Buffer Request" come back): such a capture names no kernel of ours at all, and
    it is taken again."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = " ".join(e.key for e in prof.key_averages())
        if "kgrec::" in names:
            break
    return names


def _grads(m):
    return {k: _dense(getattr(m, k + "_embeddings").weight.grad) for k in ("ent", "rel", "proj")}


# (d, l1, K, ids, grad_loss, relations, positives, batch_pos, kernel).  k_run_step_r takes d >= 32 with at least 4 groups
# per relation of the table; the others run k_group_step_r (d = 16, or short relation runs).  Every batch_pos leaves a
# partial last batch; 400-600 entities make repeated rows within a batch common.
CASES = [
    (16, False, 2, "int32", 1.0, 5, 300, 128, "k_group_step_r"),
    (16, True, 14, "int64", 0.5, 3, 203, 64, "k_group_step_r"),
    (32, True, 1, "int64", 0.5, 5, 333, 100, "k_run_step_r"),
    (32, False, 2, "int32", 1.0, 100, 211, 64, "k_group_step_r"),
    (64, True, 10, "int64", 1.0, 3, 257, 100, "k_run_step_r"),
    (100, False, 10, "int64", 1.0, 7, 403, 128, "k_run_step_r"),
    (100, True, 14, "int32", 0.5, 200, 403, 128, "k_group_step_r"),
    (100, True, 2, "int32", 0.5, 9, 517, 200, "k_run_step_r"),
    (128, False, 14, "int32", 0.5, 6, 403, 150, "k_run_step_r"),
    (128, True, 10, "int64", 1.0, 300, 257, 100, "k_group_step_r"),
    (128, False, 1, "int64", 1.0, 4, 300, 77, "k_run_step_r"),
]


def _case_id(c):
    return "d%d-%s-K%d-%s-g%s-%s" % (c[0], "l1" if c[1] else "l2", c[2], c[3], c[4], c[8][2:7])


@pytest.mark.gpu
@pytest.mark.parametrize("c", CASES, ids=_case_id)
def test_reg_step_matches_the_drivers_loss(c):
    d, l1, K, idx, gl, R, n_pos, bp, kern = c
    E = 400 if d < 100 else 600
    m = _make(d, E, R, l1, seed=d + K)
    pos, corrupt = _inputs(E, R, n_pos, K, seed=d * 7 + K, idx=idx)
    want = ref_step(m._weights(), pos, corrupt, K, bp, 1.0, l1, gl)
    # a sign flip of residual component a moves two entity rows, row a of M_r and element a of r
    budget = {"ent": 2 * d * want["n_amb"], "proj": d * want["n_amb"], "rel": want["n_amb"]}
    for gm in ("dense", "sparse"):
        m.grad_mode = gm
        m.zero_grad()
        names = _kernels_that_ran(lambda: m.loss_step_corrupt(pos, corrupt, margin=1.0, batch_pos=bp, grad_loss=gl, reg=True))
        assert kern in names and ({"k_run_step_r", "k_group_step_r"} - {kern}).pop() not in names, names
        m.zero_grad()
        sl, sp, sn = m.loss_step_corrupt(pos, corrupt, margin=1.0, batch_pos=bp, grad_loss=gl, reg=True)
        _close(sp, want["pos"], "pos", rtol=2e-5, atol_rel=1e-5)
        _close(sn, want["neg"], "neg", rtol=2e-5, atol_rel=1e-5)
        _close(sl, want["loss"], "loss", rtol=2e-5, atol_rel=1e-5)
        got = _grads(m)
        for k in ("ent", "rel", "proj"):
            _close(got[k], want[k], "%s %s" % (gm, k), max_outliers=budget[k])
    m.check_indices()


@pytest.mark.gpu
@pytest.mark.parametrize("c", [CASES[0], CASES[5], CASES[6], CASES[8]], ids=_case_id)
def test_reg_alone_when_every_hinge_is_inactive(c):
    """A margin so negative that no hinge is active: the loss is the regulariser's and so are the gradients -- non-zero
    exactly on the gathered rows outside the unit sphere, and zero on proj."""
    d, l1, K, idx, gl, R, n_pos, bp, _ = c
    E = 400 if d < 100 else 600
    m = _make(d, E, R, l1, seed=3 + d)
    pos, corrupt = _inputs(E, R, n_pos, K, seed=5 + d, idx=idx)
    want = ref_step(m._weights(), pos, corrupt, K, bp, -1e4, l1, gl)
    h, t, r, nh, nt, nr = _ids(*pos, corrupt, K)
    w = m._weights()
    outside = {k: (w[k].detach() ** 2).sum(1) > 1 for k in ("ent", "rel")}
    touched = {"ent": torch.zeros(E, dtype=torch.bool, device="cuda"), "rel": torch.zeros(R, dtype=torch.bool, device="cuda")}
    touched["ent"][torch.cat([h, t, nh, nt])] = True
    touched["rel"][r] = True
    for gm in ("dense", "sparse"):
        m.grad_mode = gm
        m.zero_grad()
        sl, _, _ = m.loss_step_corrupt(pos, corrupt, margin=-1e4, batch_pos=bp, grad_loss=gl, reg=True)
        _close(sl, want["loss"], "loss", rtol=2e-5, atol_rel=1e-5)
        got = _grads(m)
        assert not got["proj"].any()
        for k in ("ent", "rel"):
            _close(got[k], want[k], "%s %s" % (gm, k), rtol=1e-5, atol_rel=1e-6)
            nz = got[k].ne(0).any(1).cuda()
            assert torch.equal(nz, touched[k] & outside[k]), k


@pytest.mark.gpu
@pytest.mark.parametrize("c", [CASES[1], CASES[4], CASES[6], CASES[8]], ids=_case_id)
def test_reg_inactive_inside_the_unit_ball(c):
    """Every row at norm 0.9: reg=True computes exactly what reg=False does.  Scores, losses and the slot gradients
    are compared bit for bit; proj's gradient and the dense accumulators are atomic sums whose order varies from run to
    run, so those agree to float rounding."""
    d, l1, K, idx, gl, R, n_pos, bp, _ = c
    E = 400 if d < 100 else 600
    m = _make(d, E, R, l1, seed=9 + d, scale=0.9)
    pos, corrupt = _inputs(E, R, n_pos, K, seed=11 + d, idx=idx)
    for gm in ("sparse", "dense"):
        m.grad_mode = gm
        out = []
        for reg in (False, True):
            m.zero_grad()
            res = m.loss_step_corrupt(pos, corrupt, margin=1.0, batch_pos=bp, grad_loss=gl, reg=reg)
            out.append((res, {k: getattr(m, k + "_embeddings").weight.grad for k in ("ent", "rel", "proj")}))
        (a, ga), (b, gb) = out
        for x, y in zip(a, b):
            assert torch.equal(x, y)
        for k in ("ent", "rel", "proj"):
            if gm == "sparse" and k != "proj":
                assert torch.equal(ga[k]._indices(), gb[k]._indices()) and torch.equal(ga[k]._values(), gb[k]._values()), k
            else:
                torch.testing.assert_close(_dense(ga[k]), _dense(gb[k]), rtol=1e-6, atol=1e-6 * max(1.0, float(_dense(ga[k]).abs().max())))


# ---- GPU: optimizer trajectories -------------------------------------------------------------------------------------
def _traj_batch(gen, E, R, B=48, KN=2):
    pos = tuple(torch.randint(0, n, (B,), generator=gen).cuda() for n in (E, E, R))
    cid = torch.randint(0, E, (B * KN,), generator=gen, dtype=torch.int32)
    return pos, torch.where(torch.rand(B * KN, generator=gen) < 0.5, ~cid, cid).cuda()


def _torch_opt(kind, params, lr, wd, momentum):
    if kind == "SGD":
        return torch.optim.SGD(params, lr=lr, weight_decay=wd, momentum=momentum)
    if kind == "Adagrad":
        return torch.optim.Adagrad(params, lr=lr, weight_decay=wd)
    return torch.optim.Adam(params, lr=lr, weight_decay=wd)


TRAJ = [   # (optimizer, lr, weight decay, momentum, clip, L1, rows): transr.sh (Adam, L1, lr 1e-3, clip 5), momentum SGD, Adagrad
    ("Adam", 1e-3, 0.0, 0.0, 5.0, True, "all"),
    ("SGD", 1e-2, 1e-5, 0.9, 0.5, False, "all"),
    ("Adagrad", 5e-3, 0.0, 0.0, 5.0, True, "touched"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,lr,wd,momentum,clip,l1,rows", TRAJ)
def test_optimizer_trajectory_on_the_drivers_loss(kind, lr, wd, momentum, clip, l1, rows):
    """SparseRowOptimizer.step_corrupt(reg=True) for 20 steps against torch.optim + clip_grad_norm_ on float64 tables
    driven by the autograd restatement of the driver's loss (every row of every table moves on every step where the
    rule says so; rows="touched" with Adagrad, whose untouched rows a zero gradient leaves unchanged)."""
    from kgrec_b200.optim import SparseRowOptimizer
    d, E, R = 16, 1500, 9
    m = _make(d, E, R, l1, seed=31)
    ref = {k: torch.nn.Parameter(v.detach().double().clone()) for k, v in m._weights().items()}
    ropt = _torch_opt(kind, list(ref.values()), lr, wd, momentum)
    opt = SparseRowOptimizer(m, optimizer_type=kind, lr=lr, l2_lambda=wd, clip=clip, momentum=momentum, rows=rows)
    gen = torch.Generator().manual_seed(17)
    for _ in range(20):
        pos, corrupt = _traj_batch(gen, E, R)
        ropt.zero_grad()
        g = ref_step(ref, pos, corrupt, 2, pos[0].numel(), 1.0, l1, 1.0)
        for k, p in ref.items():
            p.grad = g[k].to(p.device)
        torch.nn.utils.clip_grad_norm_(list(ref.values()), clip)
        ropt.step()
        opt.step_corrupt(pos, corrupt, margin=1.0, reg=True)
    torch.cuda.synchronize()
    for k, v in m._weights().items():
        torch.testing.assert_close(v.detach().double().cpu(), ref[k].detach().cpu(), rtol=1e-4, atol=2.5e-5, msg=lambda s: "%s: %s" % (k, s))
    m.check_indices()


# ---- GPU: CUDA graphs ------------------------------------------------------------------------------------------------
N_ENT, N_REL, N_TRIPLES, BATCH, N_STEPS, D = 700, 11, 2600, 256, 25, 64       # 10 batches an epoch: 2.5 epochs


def _loop_env():
    from kgrec_b200.data import DeviceTrainIterator
    from kgrec_b200.optim import SparseRowOptimizer
    from kgrec_b200.sampling import TripleNegativeSampler
    rng = np.random.RandomState(0)
    m = _make(D, N_ENT, N_REL, True, seed=0)
    triples = np.stack([rng.randint(0, N_ENT, N_TRIPLES), rng.randint(0, N_ENT, N_TRIPLES), rng.randint(0, N_REL, N_TRIPLES)], 1)
    it = DeviceTrainIterator(triples, BATCH, device="cuda", seed=1)
    smp = TripleNegativeSampler(N_ENT, N_REL, known_triples=triples)
    opt = SparseRowOptimizer(m, optimizer_type="Adam", lr=1e-3, clip=5.0)
    return m, it, smp, opt


def _snapshot(m, opt):
    snap = {"w." + k: v.detach().clone() for k, v in m.named_parameters()}
    for name, dd in (("acc", opt.acc), ("s1", opt.s1), ("s2", opt.s2)):
        snap.update({name + "." + k: v.clone() for k, v in dd.items() if v is not None})
    return snap


@pytest.mark.gpu
def test_graphed_loop_with_reg_matches_eager_and_host_steps():
    """GraphedTrainLoop(reg=True) on TransR: 10-step graphs against the same `_dev` launches run eagerly
    (steps_per_graph=0) and against host-scalar step_corrupt(reg=True) calls with the same seeds, over 2.5 epochs."""
    from kgrec_b200.train import GraphedTrainLoop
    K = 3
    snaps = []
    for mode in (10, 0, "host"):
        m, it, smp, opt = _loop_env()
        if mode == "host":
            losses = []
            for _ in range(N_STEPS):
                s = opt.t + 1
                pos = next(it)
                out = opt.step_corrupt(pos, smp.sample(pos, K, seed=77 + s), margin=1.0, reg=True)
                losses.append(out.view(-1)[:1])
            loss = torch.cat(losses)
        else:
            loss = GraphedTrainLoop(m, opt, it, smp, K, steps_per_graph=mode, reg=True, sample_seed=77).run(N_STEPS)
        torch.cuda.synchronize()
        snap = _snapshot(m, opt)
        snap["loss"] = loss
        snaps.append((snap, it, opt))
        m.check_indices()
    (g, git, gopt), (e, _, _), (h, hit, hopt) = snaps
    for other in (e, h):
        assert g.keys() == other.keys()
        for k in g:
            torch.testing.assert_close(g[k], other[k], rtol=2e-5, atol=2e-5, msg=lambda s: "%s: %s" % (k, s))
    assert (git.start, git.epoch) == (hit.start, hit.epoch) and git.epoch >= 2
    assert gopt.t == hopt.t == N_STEPS


@pytest.mark.gpu
@pytest.mark.parametrize("grad_mode", ["sparse", "dense"])
def test_graphed_loss_step_with_reg_equals_the_direct_call(grad_mode):
    d, l1, K, idx, gl, R, n_pos, bp, _ = CASES[5]
    E = 600
    m = _make(d, E, R, l1, seed=2)
    m.grad_mode = grad_mode
    pos, corrupt = _inputs(E, R, n_pos, K, seed=4, idx="int32")
    step = m.graphed_loss_step(n_pos, K, margin=1.0, batch_pos=bp, grad_loss=gl, reg=True)
    step.h.copy_(pos[0]), step.t.copy_(pos[1]), step.r.copy_(pos[2]), step.corrupt.copy_(corrupt)
    step.replay()
    torch.cuda.synchronize()
    m.zero_grad()
    sl, sp, sn = m.loss_step_corrupt(pos, corrupt, margin=1.0, batch_pos=bp, grad_loss=gl, reg=True)
    assert torch.equal(step.loss, sl) and torch.equal(step.pos_scores, sp) and torch.equal(step.neg_scores, sn)
    got = _grads(m)
    for k in ("ent", "rel", "proj"):
        torch.testing.assert_close(_dense(step.grads[k]), got[k], rtol=1e-6, atol=1e-6 * max(1.0, float(got[k].abs().max())))
