#!/usr/bin/env python
"""Cost of the fused normLoss terms in TransR's step kernels (kgrec_corrupt_loss_step, reg_flags = 1), and the seeded
reg = False outputs to compare two builds with.

    python tools/transr_reg_step.py [--rounds 5]        one JSON line: the card, then (a) and (b)
    python tools/transr_reg_step.py --dump DIR           (c) only: DIR/transr_reg_off.npz
    python tools/transr_reg_step.py --compare A.npz B.npz

(a) the step kernel at bench.py's train_transr shape (d = 100, 100k entities, 500 relations, 32 batches of 1024
    positives x 10 negatives, L2): graphed_loss_step replays (counting sort by relation + k_run_step_r + batch losses),
    reg off and on alternated `--rounds` times, CUDA events; gradients dense (what SparseRowOptimizer accumulates) and
    in slots.  Tables at norm 1.05 / 0.95 alternating ("half": half the rows carry the regulariser) and all at 1.05
    ("all": every row does, the most the regulariser can cost).
(b) GraphedTrainLoop per-batch steps at transr.sh's shape (batch 256, d = 100, L1, 1 negative, Adam lr 1e-3, clip 5;
    40k entities, 200 relations, 200k triples), 10-step graphs, rows="touched" and "all", reg off and on.
(c) scores, per-batch losses and gradients of reg = False steps on seeded inputs, for both TransR step kernels
    (k_run_step_r: 7 relations; k_group_step_r: 500 relations) in both gradient modes.  Scores and losses of two builds
    should be bit-identical; slot gradients of ent / rel too; proj and dense gradients are atomic sums and agree up to
    their order.
There is no CPU fallback.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "joint-kg-recommender_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def scaled(m, half):
    with torch.no_grad():
        for tab in (m.ent_embeddings.weight, m.rel_embeddings.weight):
            n = tab.shape[0]
            s = torch.where(torch.arange(n, device=tab.device) % 2 == 0, 1.05, 0.95) if half else torch.full((n,), 1.05, device=tab.device)
            tab.mul_(s.view(-1, 1) / tab.norm(dim=1, keepdim=True))
    return m


def corrupt_ids(gen, n_pos, k, n_ent):
    cid = torch.randint(0, n_ent, (n_pos * k,), generator=gen, dtype=torch.int32)
    return torch.where(torch.rand(n_pos * k, generator=gen) < 0.5, ~cid, cid)


def kernel_cost(rounds):
    """(a): ms per graphed step launch, reg off / on alternated."""
    import kgrec_b200 as K
    from kgrec_b200.models.base import device_init
    d, n_ent, n_rel, k, n_pos = 100, 100_000, 500, 10, 32 * 1024
    dev = torch.device("cuda")
    gen = torch.Generator().manual_seed(0)
    ids = [torch.randint(0, n, (n_pos,), generator=gen, dtype=torch.int32).to(dev) for n in (n_ent, n_ent, n_rel)]
    corrupt = corrupt_ids(gen, n_pos, k, n_ent).to(dev)
    out = {}
    for rows in ("half", "all"):
        torch.manual_seed(0)
        with device_init(dev):
            m = scaled(K.TransRModel(False, d, n_ent, n_rel), rows == "half")
        for gm in ("dense", "sparse"):
            m.grad_mode = gm
            steps = {}
            for reg in (False, True):
                s = m.graphed_loss_step(n_pos, k, margin=1.0, batch_pos=1024, reg=reg)
                s.h.copy_(ids[0]), s.t.copy_(ids[1]), s.r.copy_(ids[2]), s.corrupt.copy_(corrupt)
                steps[reg] = s
            ms = {False: [], True: []}
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            for s in steps.values():
                for _ in range(3):
                    s.replay()
            for _ in range(rounds):
                for reg, s in steps.items():
                    torch.cuda.synchronize()
                    a.record()
                    for _ in range(20):
                        s.replay()
                    b.record()
                    torch.cuda.synchronize()
                    ms[reg].append(a.elapsed_time(b) / 20)
            off, on = min(ms[False]), min(ms[True])
            out["%s_rows_%s" % (rows, gm)] = {"ms_reg_off": ms[False], "ms_reg_on": ms[True], "best_ratio_on_off": on / off}
            del steps
        m.check_indices()
        del m
    return out


def loop_cost(steps):
    """(b): µs per GraphedTrainLoop step."""
    import kgrec_b200 as K
    from kgrec_b200.data import DeviceTrainIterator
    from kgrec_b200.models.base import device_init
    from kgrec_b200.optim import SparseRowOptimizer
    from kgrec_b200.sampling import TripleNegativeSampler
    from kgrec_b200.train import GraphedTrainLoop
    out = {}
    for rows in ("touched", "all"):
        for reg in (False, True):
            rng = np.random.RandomState(0)
            torch.manual_seed(0)
            t = np.stack([rng.randint(0, 40_000, 200_000), rng.randint(0, 40_000, 200_000), rng.randint(0, 200, 200_000)], 1)
            with device_init(torch.device("cuda")):
                m = K.TransRModel(True, 100, 40_000, 200)
            it = DeviceTrainIterator(t, 256, seed=1)
            opt = SparseRowOptimizer(m, "Adam", lr=1e-3, clip=5.0, rows=rows)
            loop = GraphedTrainLoop(m, opt, it, TripleNegativeSampler(40_000, 200, known_triples=t), 1, steps_per_graph=10, reg=reg)
            loop.run(steps)                    # warm-up: captures, allocator
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            loop.run(steps)
            b.record()
            torch.cuda.synchronize()
            m.check_indices()
            out["%s_reg_%s" % (rows, "on" if reg else "off")] = {"us_per_step": a.elapsed_time(b) * 1e3 / steps}
    return out


def dump(path):
    """(c)."""
    import kgrec_b200 as K
    os.makedirs(path, exist_ok=True)
    res = {}
    for name, n_rel in (("run", 7), ("group", 500)):
        for gm in ("dense", "sparse"):
            torch.manual_seed(1)
            m = scaled(K.TransRModel(False, 100, 2000, n_rel), True)
            m.grad_mode = gm
            gen = torch.Generator().manual_seed(2)
            n_pos, k = 1500, 10
            pos = tuple(torch.randint(0, n, (n_pos,), generator=gen).cuda() for n in (2000, 2000, n_rel))
            corrupt = corrupt_ids(gen, n_pos, k, 2000).cuda()
            lo, ps, ns = m.loss_step_corrupt(pos, corrupt, margin=1.0, batch_pos=256)
            key = "%s_%s_" % (name, gm)
            res[key + "loss"], res[key + "pos"], res[key + "neg"] = (x.cpu().numpy() for x in (lo, ps, ns))
            for tab in ("ent", "rel", "proj"):
                g = getattr(m, tab + "_embeddings").weight.grad
                if g.is_sparse:
                    res[key + tab + "_slots"] = g._values().cpu().numpy()
                    res[key + tab + "_ids"] = g._indices().cpu().numpy()
                    g = g.to_dense()
                res[key + tab] = g.cpu().numpy()
            m.check_indices()
    np.savez(os.path.join(path, "transr_reg_off.npz"), **res)
    print(json.dumps({"dumped": os.path.join(path, "transr_reg_off.npz"), "arrays": len(res)}))


def compare(a, b):
    A, B = np.load(a), np.load(b)
    out = {}
    for k in sorted(A.files):
        x, y = A[k], B[k]
        same = x.shape == y.shape and np.array_equal(x.view(np.uint8), y.view(np.uint8))
        out[k] = "bit-identical" if same else "max |diff| %.3g (max |x| %.3g)" % (np.abs(x.astype(np.float64) - y).max(), np.abs(x).max())
    print(json.dumps(out, indent=1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--loop-steps", type=int, default=400)
    ap.add_argument("--dump", metavar="DIR")
    ap.add_argument("--compare", nargs=2, metavar="NPZ")
    a = ap.parse_args()
    if a.compare:
        return compare(*a.compare)
    if a.dump:
        return dump(a.dump)
    from step_e_floor import gpu_info
    out = {"gpu": gpu_info(), "step_kernel_bench_shape": kernel_cost(a.rounds), "graphed_loop_transr_sh": loop_cost(a.loop_steps)}
    out["gpu_after"] = gpu_info()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
