#!/usr/bin/env python
"""Training rate with the reference's semantics -- one optimizer update per batch of 1024 positives -- eagerly and
replayed from CUDA graphs.

    python tools/train_loop_graph.py [--steps 400] [--graphs 1,10,100]

Prints ONE JSON line.  Per workload, steps/s and positives/s of
  eager   the loop of INTEGRATION section 6: next(DeviceTrainIterator) -> sampler.sample -> SparseRowOptimizer.step_*
  S=<n>   GraphedTrainLoop.run with steps_per_graph n (KTUP: n rounded up to its 10-step cycle)
over --steps steps after a warm-up of the same length (graph capture included there), CUDA events around the
whole run.  Workloads, all at d = 100, Adagrad lr 0.005, clip 5:
  transe_k1 / transe_k10   TransE L1, 40k entities, 200 relations, 200k triples, 1 / 10 negatives
  transh_reg               TransH L1 with normLoss + orthogonalLoss, 1 negative
  transr                   TransR L2, 1 negative
  tup_soft / tup_gumbel    TUP L2, 6040 users x 3706 items, P = 20, 1M ratings, 1 negative item
  ktup_cycle               KTUP configs[3] shapes (6040 x 3706, 500k entities, R = P = 20), joint_ratio 0.5, reg
The card name, power limit and clocks are read in the same call.  There is no CPU fallback.
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

from step_e_floor import gpu_info  # noqa: E402

D, BATCH = 100, 1024


def make(name):
    import kgrec_b200 as K
    from kgrec_b200.data import DeviceTrainIterator
    from kgrec_b200.models.base import device_init
    from kgrec_b200.optim import SparseRowOptimizer
    from kgrec_b200.sampling import RatingNegativeSampler, TripleNegativeSampler
    rng = np.random.RandomState(0)
    torch.manual_seed(0)
    dev = torch.device("cuda")
    w = {"name": name, "n_neg": 10 if name == "transe_k10" else 1, "reg": name in ("transh_reg", "ktup_cycle")}

    def triples(n_ent, n_rel, n):
        return np.stack([rng.randint(0, n_ent, n), rng.randint(0, n_ent, n), rng.randint(0, n_rel, n)], 1)

    def ratings(n):
        return np.stack([rng.randint(0, 6040, n), rng.randint(0, 3706, n)], 1)
    with device_init(dev):
        if name.startswith(("transe", "transh", "transr")):
            cls = {"e": K.TransEModel, "h": K.TransHModel, "r": K.TransRModel}[name[5]]
            w["model"] = cls(name != "transr", D, 40_000, 200)
            t = triples(40_000, 200, 200_000)
            w["it"] = DeviceTrainIterator(t, BATCH, seed=1)
            w["sampler"] = TripleNegativeSampler(40_000, 200, known_triples=t)
        elif name.startswith("tup"):
            w["model"] = K.TransUPModel(False, D, 6040, 3706, 20, name == "tup_gumbel")
            r = ratings(1_000_000)
            w["it"] = DeviceTrainIterator(r, BATCH, seed=1)
            w["sampler"] = RatingNegativeSampler(3706, known_ratings=r)
        else:
            ents = rng.permutation(500_000)[:3706]
            new_map = {i: (int(ents[i]) if i % 10 < 7 else -1, i) for i in range(3706)}
            w["model"] = K.jTransUPModel(False, D, 6040, 3706, 500_000, 20, {i: i for i in range(3706)}, new_map, False, False)
            r, t = ratings(1_000_000), triples(500_000, 20, 2_000_000)
            w["it"] = DeviceTrainIterator(r, BATCH, seed=1)
            w["sampler"] = RatingNegativeSampler(3706, known_ratings=r)
            w["kg_it"] = DeviceTrainIterator(t, BATCH, seed=2)
            w["kg_sampler"] = TripleNegativeSampler(500_000, 20, known_triples=t)
    w["opt"] = SparseRowOptimizer(w["model"], "Adagrad", lr=0.005, clip=5.0)
    return w


def eager_runner(w):
    opt, ktup = w["opt"], "kg_it" in w
    rec = w["name"].startswith("tup")
    cnt = [0]

    def run(n):
        for _ in range(n):
            g = cnt[0]
            cnt[0] += 1
            if rec or (ktup and g % 10 < 5):
                u, i = next(w["it"])
                ni = w["sampler"].sample(u, i, w["n_neg"], seed=g)
                opt.step_pairs((u, i), (u, ni), target=-1.0, reg=w["reg"])
            else:
                it, smp = (w["kg_it"], w["kg_sampler"]) if ktup else (w["it"], w["sampler"])
                pos = next(it)
                opt.step_corrupt(pos, smp.sample(pos, w["n_neg"], seed=g), margin=1.0, reg=w["reg"])
    return run


def graph_runner(w, S):
    from kgrec_b200.train import GraphedTrainLoop
    kw = dict(steps_per_graph=S, reg=w["reg"])
    if "kg_it" in w:
        kw.update(kg_iterator=w["kg_it"], kg_sampler=w["kg_sampler"], joint_ratio=0.5, kg_lambda=1.0)
    loop = GraphedTrainLoop(w["model"], w["opt"], w["it"], w["sampler"], w["n_neg"], **kw)
    return loop.run


def timed(run, steps):
    run(steps)                      # warm-up: captures, allocator, clocks
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    run(steps)
    b.record()
    torch.cuda.synchronize()
    ms = a.elapsed_time(b)
    return {"steps_per_s": steps / (ms * 1e-3), "positives_per_s": steps * BATCH / (ms * 1e-3), "us_per_step": ms * 1e3 / steps}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=400)
    ap.add_argument("--graphs", default="1,10,100")
    ap.add_argument("--workloads", default="transe_k1,transe_k10,transh_reg,transr,tup_soft,tup_gumbel,ktup_cycle")
    a = ap.parse_args()
    info = gpu_info()
    out = {"batch_size": BATCH, "d": D, "steps": a.steps}
    for name in a.workloads.split(","):
        res = {"eager": timed(eager_runner(make(name)), a.steps)}
        for S in (int(s) for s in a.graphs.split(",")):
            S_eff = S if name != "ktup_cycle" or S <= 1 else -(-S // 10) * 10
            res["S=%d" % S_eff] = timed(graph_runner(make(name), S_eff), a.steps)
        res["graph_speedup_max"] = max(v["steps_per_s"] for k, v in res.items() if k.startswith("S=")) / res["eager"]["steps_per_s"]
        out[name] = res
    out["gpu"] = info
    out["gpu_after"] = gpu_info()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
