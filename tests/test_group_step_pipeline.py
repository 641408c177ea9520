"""The main loop of the TMA-staged TransE step kernel (k_group_step_e_tma): ids loaded a group ahead, all rows of a group
read before its stage is refilled, one reduce-scatter for the 1 + K scores, coefficients in lanes.

Every case runs on the TMA side of the dispatch (sparse slot gradients, no fused regulariser, ring within 225 KB, at least
two groups per warp) and is compared bit for bit -- losses, positive and negative scores, every slot value and the COO
ids -- with the register kernel k_group_step_e, run on the same inputs cut at batch boundaries into launches too small
for the TMA kernel.  The cases cover:
  * 1 + K <= 16 (the 16-slot reduce-scatter, rows kept in registers), 1 + K = 17 (the 32-slot reduce-scatter crosses
    a half-warp) and K = 29 (the largest K this kernel takes; rows read twice);
  * d in {4, 36, 100, 128}, L1 and L2, margin and BPR, int32 and int64 ids;
  * a launch whose last CTA gets fewer groups than the others, and the smallest launch the dispatch sends here.
One more test puts an out-of-range id in a batch: the kernel clamps it, raises the status word and does not fault.
"""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "joint-kg-recommender_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

pytestmark = pytest.mark.gpu

BATCH_POS, N_ENT, N_REL = 100, 3000, 23
WARPS, STAGES = 16, 2       # kTmaWarps, kTmaStages


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def smallest_launch():
    """The fewest positives the dispatch still sends to the TMA kernel: two groups per warp on every SM."""
    return 2 * WARPS * sm_count()


def ring_fits(d, k):
    return ((WARPS * STAGES * 136 + 127) & ~127) + WARPS * STAGES * (3 + k) * d * 4 <= 225 * 1024


# (d, K, L1, loss, index dtype, n_pos): n_pos "partial" = two groups per warp plus a few, so the grid-stride loop
# leaves the last warps and CTAs with fewer groups; "min" = the smallest launch on the TMA kernel
CASES = [
    (100, 10, False, "margin", "int32", "partial"),
    (100, 10, True, "bpr", "int64", "min"),
    (128, 10, False, "bpr", "int64", "partial"),
    (128, 1, True, "margin", "int32", "min"),
    (100, 14, True, "margin", "int32", "partial"),
    (36, 15, False, "margin", "int64", "partial"),
    (4, 15, True, "bpr", "int32", "partial"),
    (36, 16, False, "margin", "int32", "partial"),
    (4, 16, True, "bpr", "int64", "min"),
    (36, 16, True, "margin", "int64", "min"),
    (36, 29, False, "bpr", "int32", "partial"),
    (4, 29, False, "margin", "int64", "partial"),
    (36, 29, True, "margin", "int32", "min"),
    (4, 29, True, "bpr", "int64", "partial"),
]
assert all(ring_fits(c[0], c[1]) for c in CASES)
assert {(c[2], c[3]) for c in CASES} == {(False, "margin"), (True, "margin"), (False, "bpr"), (True, "bpr")}


def case_id(c):
    d, k, l1, loss, idt, npos = c
    return "d%d-k%d-%s-%s-%s-%s" % (d, k, "l1" if l1 else "l2", loss, idt, npos)


def n_pos_of(c):
    return smallest_launch() + (37 if c[5] == "partial" else 0)


def make_inputs(c, seed):
    d, k, l1, loss, idt, _ = c
    n_pos = n_pos_of(c)
    g = torch.Generator().manual_seed(seed)
    dt = torch.int32 if idt == "int32" else torch.int64
    h = torch.randint(0, N_ENT, (n_pos,), generator=g, dtype=dt)
    t = torch.randint(0, N_ENT, (n_pos,), generator=g, dtype=dt)
    r = torch.randint(0, N_REL, (n_pos,), generator=g, dtype=dt)
    cid = torch.randint(0, N_ENT, (n_pos * k,), generator=g, dtype=torch.int32)
    head = torch.rand(n_pos * k, generator=g) < 0.5
    return h, t, r, cid, torch.where(head, ~cid, cid)


def slices(n_pos):
    """[lo, hi) ranges of whole loss batches, each of fewer positives than the smallest TMA launch."""
    step = (smallest_launch() - 1) // BATCH_POS * BATCH_POS
    return [(lo, min(n_pos, lo + step)) for lo in range(0, n_pos, step)]


def run_case(c, rows=None):      # rows = (j0, j1): only positives j0 .. j1 - 1 (whole batches) and their negatives
    import kgrec_b200 as K
    d, k, l1, loss, _, _ = c
    seed = 2000 + CASES.index(c)
    torch.manual_seed(seed)
    m = K.TransEModel(l1, d, N_ENT, N_REL)
    m.grad_mode = "sparse"
    h, t, r, cid, corrupt = make_inputs(c, seed)
    j0, j1 = rows if rows is not None else (0, h.numel())
    param = 1.0 if loss == "margin" else 0.5
    kw = {"margin": param} if loss == "margin" else {"loss": "bpr", "margin": param}
    lo, ps, ns = m.loss_step_corrupt(tuple(x[j0:j1].cuda() for x in (h, t, r)), corrupt[j0 * k:j1 * k].cuda(),
                                     batch_pos=BATCH_POS, **kw)
    m.check_indices()
    torch.cuda.synchronize()
    out = {"loss": lo, "pos": ps, "neg": ns}
    for name in ("ent", "rel"):
        gs = getattr(m, name + "_embeddings").weight.grad
        out[name] = gs._values()
        out[name + "_ids"] = gs._indices()
    return {key: v.cpu().numpy() for key, v in out.items()}, (h, t, r, cid)


@pytest.fixture(scope="module")
def register_values():
    """Every output of k_group_step_e for every case: a group's slot values and scores do not depend on the launch, and
    slices of whole batches keep each batch's loss (BPR's per-batch count included), so the slices concatenated are
    the outputs of the whole case."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):          # a capture whose kernel records the profiler lost names no kernel of ours: take it again
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run_case(CASES[0], slices(n_pos_of(CASES[0]))[0])
            torch.cuda.synchronize()
        names = " ".join(e.key for e in prof.key_averages())
        if "kgrec::" in names:
            break
    assert "k_group_step_e" in names and "k_group_step_e_tma" not in names, names
    out = {}
    for c in CASES:
        parts = [run_case(c, rows)[0] for rows in slices(n_pos_of(c))]
        out[case_id(c)] = {key: np.concatenate([p[key] for p in parts], axis=1 if key.endswith("_ids") else 0)
                           for key in parts[0]}
    return out


@pytest.mark.parametrize("c", CASES, ids=case_id)
def test_pipeline_matches_register_kernel(c, register_values):
    k = c[1]
    got, (h, t, r, cid) = run_case(c)
    for key, v in got.items():
        want = register_values[case_id(c)][key]
        assert v.shape == want.shape and v.dtype == want.dtype, key
        assert np.array_equal(v.view(np.uint8), want.view(np.uint8)), key
    want_ent = torch.cat([h.long().view(-1, 1), t.long().view(-1, 1), cid.long().view(-1, k)], dim=1).view(1, -1)
    assert np.array_equal(got["ent_ids"], want_ent.numpy())
    assert np.array_equal(got["rel_ids"], r.long().view(1, -1).numpy())


def test_pipeline_kernel_is_the_one_that_runs():
    """The cases above reach k_group_step_e_tma (named in a profile), and one positive fewer than the smallest
    launch does not."""
    import kgrec_b200 as K
    from torch.profiler import ProfilerActivity, profile
    c = (100, 10, False, "margin", "int32", "min")
    h, t, r, _, corrupt = make_inputs(c, 7)
    m = K.TransEModel(False, 100, N_ENT, N_REL)
    m.grad_mode = "sparse"
    names = []
    for n in (smallest_launch(), smallest_launch() - 1):
        dev = [x[:n].cuda() for x in (h, t, r)] + [corrupt[: n * c[1]].cuda()]
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            m.loss_step_corrupt(tuple(dev[:3]), dev[3], batch_pos=BATCH_POS, margin=1.0)
            torch.cuda.synchronize()
        names.append(" ".join(e.key for e in prof.key_averages()))
    m.check_indices()
    assert "k_group_step_e_tma" in names[0]
    assert "k_group_step_e_tma" not in names[1] and "k_group_step_e" in names[1]


@pytest.mark.parametrize("where", ["corrupt", "head", "relation"])
def test_pipeline_out_of_range_id_raises_status(where):
    """One id past its table: clamped to row 0 and reported by the status word; the launch completes."""
    import kgrec_b200 as K
    c = (100, 10, False, "margin", "int64", "partial")
    h, t, r, cid, corrupt = make_inputs(c, 11)
    j = n_pos_of(c) - 3          # a group in the last round of the grid-stride loop
    if where == "corrupt":
        corrupt[j * c[1] + 4] = N_ENT + 5
    elif where == "head":
        h[j] = N_ENT
    else:
        r[j] = N_REL + 1
    m = K.TransEModel(False, 100, N_ENT, N_REL)
    m.grad_mode = "sparse"
    lo, ps, ns = m.loss_step_corrupt(tuple(x.cuda() for x in (h, t, r)), corrupt.cuda(), batch_pos=BATCH_POS, margin=1.0)
    torch.cuda.synchronize()
    with pytest.raises(IndexError):
        m.check_indices()
    m.check_indices()            # the word was cleared by the raise
    assert bool(torch.isfinite(lo).all()) and bool(torch.isfinite(ps).all()) and bool(torch.isfinite(ns).all())
