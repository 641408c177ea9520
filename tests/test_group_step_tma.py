"""The TMA-staged TransE step kernel (k_group_step_e_tma, 16 warps x 2 stages): slot gradients at d <= 128 without the
fused regulariser whenever its ring fits in shared memory; k_group_step_e otherwise and for dense accumulation.

Every case runs 5017 positives (enough for two groups per warp on 132 SMs; the last CTA's share is partial) in loss
batches of 100 (not aligned to the 16 groups a CTA takes at a time) and checks, for the sparse-mode call:
  * losses, positive and negative scores are bit for bit those of the dense-mode call (k_group_step_e, same process);
  * the densified gradients match the dense-mode gradients (atomics there: equal up to the order of the sums);
  * the COO row ids are [h, t, corrupted_1..K] per group and r per group;
  * without the fused regulariser, the slot values are bit for bit those of the register kernel k_group_step_e, run on
    the same inputs cut at batch boundaries into launches too small for the TMA kernel.
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

N_POS, BATCH_POS, N_ENT, N_REL = 5017, 100, 3000, 23


def kernel_side(d, k, reg):
    """Which kernel the dispatch picks for sparse slot gradients: 16 warps x 2 stages of (3 + K) rows (+ 136 B of
    barriers and ids) within 225 KB of shared memory, at most 29 negatives, no fused regulariser (and at least two
    groups per warp: N_POS >= 2 x 16 x 132 SMs)."""
    smem = ((16 * 2 * 136 + 127) & ~127) + 16 * 2 * (3 + k) * d * 4
    return "tma" if (not reg and k <= 29 and smem <= 225 * 1024) else "register"


def cases():
    out = []
    combos = [(False, "margin"), (True, "margin"), (False, "bpr"), (True, "bpr")]
    i = 0
    for d in (4, 64, 100, 128):
        for k in (1, 2, 10, 13, 31, 32):
            l1, loss = combos[i % 4]
            out.append((d, k, l1, loss, False))
            out.append((d, k, not l1, "margin", True))
            i += 1
    return out


CASES = cases()
assert {kernel_side(*c[:2], c[4]) for c in CASES if not c[4]} == {"tma", "register"}


def case_id(c):
    d, k, l1, loss, reg = c
    return "d%d-k%d-%s-%s%s-%s" % (d, k, "l1" if l1 else "l2", loss, "-withreg" if reg else "", kernel_side(d, k, reg))


def slices(n_pos):
    """[lo, hi) ranges of whole loss batches, each of fewer positives than the smallest TMA launch (2 x 16 x SMs)."""
    step = (2 * 16 * torch.cuda.get_device_properties(0).multi_processor_count - 1) // BATCH_POS * BATCH_POS
    return [(lo, min(n_pos, lo + step)) for lo in range(0, n_pos, step)]


def run_case(c, mode, rows=None):
    """Case c in grad mode `mode`; `rows` = (lo, hi): only positives lo .. hi - 1 (whole batches) and their negatives."""
    import kgrec_b200 as K
    d, k, l1, loss, reg = c
    seed = 1000 + CASES.index(c)
    torch.manual_seed(seed)
    m = K.TransEModel(l1, d, N_ENT, N_REL)
    m.grad_mode = mode
    g = torch.Generator().manual_seed(seed)
    h = torch.randint(0, N_ENT, (N_POS,), generator=g, dtype=torch.int32)
    t = torch.randint(0, N_ENT, (N_POS,), generator=g, dtype=torch.int32)
    r = torch.randint(0, N_REL, (N_POS,), generator=g, dtype=torch.int32)
    cid = torch.randint(0, N_ENT, (N_POS * k,), generator=g, dtype=torch.int32)
    head = torch.rand(N_POS * k, generator=g) < 0.5
    corrupt = torch.where(head, ~cid, cid)
    dev = [x.cuda() for x in (h, t, r, corrupt)]
    if rows is not None:
        j0, j1 = rows
        dev = [x[j0:j1] for x in dev[:3]] + [dev[3][j0 * k:j1 * k]]
    param = 1.0 if loss == "margin" else 0.5
    kw = {"margin": param} if loss == "margin" else {"loss": "bpr", "margin": param}
    lo, ps, ns = m.loss_step_corrupt(tuple(dev[:3]), dev[3], batch_pos=BATCH_POS, reg=reg, **kw)
    m.check_indices()
    torch.cuda.synchronize()
    return m, (lo, ps, ns), (h, t, r, cid)


@pytest.fixture(scope="module")
def register_values():
    """Slot values of k_group_step_e for every case without the fused regulariser: a group's slot values do not depend
    on the launch, and slices of whole batches keep each batch's BPR count, so the slices concatenated are the values
    of the whole case."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):          # a capture whose kernel records the profiler lost names no kernel of ours: take it again
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run_case(CASES[0], "sparse", slices(N_POS)[0])      # CASES[0] runs on the TMA kernel when whole
            torch.cuda.synchronize()
        names = " ".join(e.key for e in prof.key_averages())
        if "kgrec::" in names:
            break
    assert "k_group_step_e" in names and "k_group_step_e_tma" not in names, names
    out = {}
    for c in (c for c in CASES if not c[4]):
        ms = [run_case(c, "sparse", rows)[0] for rows in slices(N_POS)]
        out[case_id(c)] = {name: np.concatenate([getattr(m, name + "_embeddings").weight.grad._values().cpu().numpy()
                                                 for m in ms]) for name in ("ent", "rel")}
    return out


@pytest.mark.parametrize("c", CASES, ids=case_id)
def test_tma_step_matches_register_kernels(c, register_values):
    d, k, l1, loss, reg = c
    ms, out_s, (h, t, r, cid) = run_case(c, "sparse")
    md, out_d, _ = run_case(c, "dense")
    for a, b, name in zip(out_s, out_d, ("loss", "pos_scores", "neg_scores")):
        assert torch.equal(a, b), name
    for name in ("ent", "rel"):
        gs = getattr(ms, name + "_embeddings").weight.grad
        gd = getattr(md, name + "_embeddings").weight.grad
        assert gs.is_sparse and not gd.is_sparse
        dense = gs.to_dense()
        scale = float(gd.abs().max())
        assert torch.allclose(dense, gd, rtol=1e-6, atol=1e-6 * max(scale, 1e-30)), name
    want_ent = torch.cat([h.long().view(-1, 1), t.long().view(-1, 1), cid.long().view(-1, k)], dim=1).view(1, -1)
    assert torch.equal(ms.ent_embeddings.weight.grad._indices().cpu(), want_ent)
    assert torch.equal(ms.rel_embeddings.weight.grad._indices().cpu(), r.long().view(1, -1))
    if not reg:
        for name in ("ent", "rel"):
            got = getattr(ms, name + "_embeddings").weight.grad._values().cpu().numpy()
            want = register_values[case_id(c)][name]
            assert got.shape == want.shape and np.array_equal(got.view(np.uint32), want.view(np.uint32)), name
