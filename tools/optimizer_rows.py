#!/usr/bin/env python
"""Cost of the reference's dense optimizer semantics (SparseRowOptimizer rows="all") against the O(batch) default
(rows="touched") and against torch's own dense path, at batch 1024, d = 100.

    python tools/optimizer_rows.py --leg steps [--steps 300] [--rounds 2]
    python tools/optimizer_rows.py --leg sweep [--iters 50]          (a separate run: torch.profiler on)

Each prints ONE JSON line with the card name, power limit and clocks read in the same run.  Workloads:
  transe_adam    configs[1]: TransE L1, 100k entities, 500 relations, 1 negative; Adam lr 1e-3 (transe.sh)
  tup_adagrad    configs[2] shapes: TUP, 50k users x 50k items, P = 20, soft preferences; Adagrad lr 5e-3, wd 1e-5
                 (transup.sh)
  ktup_adam      configs[3]: KTUP 6040 users x 3706 items, 500k entities, R = P = 20, joint ratio 0.5; Adam lr 1e-3
                 (ktup.sh)
All clip at 5.0.  Legs:
  steps   GraphedTrainLoop (10-step graphs) us per step with rows="touched" and rows="all", and torch's dense path --
          grad_mode="dense" copies, clip_grad_norm_(foreach=True), torch.optim with fused=True (Adam) / foreach=True
          (Adagrad) -- us per step, eager.  The configurations are alternated, --rounds times, after a warm-up of each.
  sweep   kernel time of the ALL sweep (k_rows_update_all, from torch.profiler) on one step's marks, per workload and
          table set (KTUP: its rec and KG calls), with achieved GB/s in algorithmic bytes: every row reads and writes p
          and the rule's state, a marked row also reads and clears its accumulator, 4 B of marks per row of a marked
          table.  Reported as a fraction of 3.35 TB/s (the H100 SXM data sheet).
There is no CPU fallback.
"""
import argparse
import copy
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

D, BATCH, PEAK = 100, 1024, 3.35e12
WORK = {"transe_adam": ("Adam", 1e-3, 0.0), "tup_adagrad": ("Adagrad", 5e-3, 1e-5), "ktup_adam": ("Adam", 1e-3, 0.0)}


def make(name, rows):
    import kgrec_b200 as K
    from kgrec_b200.data import DeviceTrainIterator
    from kgrec_b200.models.base import device_init
    from kgrec_b200.optim import SparseRowOptimizer
    from kgrec_b200.sampling import RatingNegativeSampler, TripleNegativeSampler
    rng = np.random.RandomState(0)
    torch.manual_seed(0)
    w = {"name": name}

    def triples(n_ent, n_rel, n):
        return np.stack([rng.randint(0, n_ent, n), rng.randint(0, n_ent, n), rng.randint(0, n_rel, n)], 1)

    def ratings(n_user, n_item, n):
        return np.stack([rng.randint(0, n_user, n), rng.randint(0, n_item, n)], 1)
    with device_init(torch.device("cuda")):
        if name == "transe_adam":
            w["model"] = K.TransEModel(True, D, 100_000, 500)
            t = triples(100_000, 500, 500_000)
            w["it"], w["sampler"] = DeviceTrainIterator(t, BATCH, seed=1), TripleNegativeSampler(100_000, 500, known_triples=t)
        elif name == "tup_adagrad":
            w["model"] = K.TransUPModel(True, D, 50_000, 50_000, 20, False)
            r = ratings(50_000, 50_000, 1_000_000)
            w["it"], w["sampler"] = DeviceTrainIterator(r, BATCH, seed=1), RatingNegativeSampler(50_000, known_ratings=r)
        else:
            ents = rng.permutation(500_000)[:3706]
            new_map = {i: (int(ents[i]) if i % 10 < 7 else -1, i) for i in range(3706)}
            w["model"] = K.jTransUPModel(True, D, 6040, 3706, 500_000, 20, {i: i for i in range(3706)}, new_map, False, False)
            r, t = ratings(6040, 3706, 1_000_000), triples(500_000, 20, 2_000_000)
            w["it"], w["sampler"] = DeviceTrainIterator(r, BATCH, seed=1), RatingNegativeSampler(3706, known_ratings=r)
            w["kg_it"] = DeviceTrainIterator(t, BATCH, seed=2)
            w["kg_sampler"] = TripleNegativeSampler(500_000, 20, known_triples=t)
    kind, lr, wd = WORK[name]
    w["opt"] = SparseRowOptimizer(w["model"], kind, lr=lr, l2_lambda=wd, clip=5.0, rows=rows)
    return w


def graph_runner(w):
    from kgrec_b200.train import GraphedTrainLoop
    kw = dict(steps_per_graph=10)
    if "kg_it" in w:
        kw.update(kg_iterator=w["kg_it"], kg_sampler=w["kg_sampler"], joint_ratio=0.5, kg_lambda=1.0)
    return GraphedTrainLoop(w["model"], w["opt"], w["it"], w["sampler"], 1, **kw).run


def dense_runner(w):
    """torch's path at the same shapes: dense-gradient copy, clip_grad_norm_, torch.optim (fused Adam / foreach Adagrad)."""
    m = copy.deepcopy(w["model"])
    m.grad_mode = "dense"
    kind, lr, wd = WORK[w["name"]]
    params = list(m.parameters())
    opt = torch.optim.Adam(params, lr=lr, weight_decay=wd, fused=True) if kind == "Adam" else \
        torch.optim.Adagrad(params, lr=lr, weight_decay=wd, foreach=True)
    ktup = "kg_it" in w
    cnt = [0]

    def run(n):
        for _ in range(n):
            g = cnt[0]
            cnt[0] += 1
            opt.zero_grad()
            if w["name"] == "tup_adagrad" or (ktup and g % 10 < 5):
                u, i = next(w["it"])
                ni = w["sampler"].sample(u, i, 1, seed=g)
                loss, _, _ = m.rank_loss((u, i), (u, ni), target=-1.0)
                loss.sum().backward()
            else:
                it, smp = (w["kg_it"], w["kg_sampler"]) if ktup else (w["it"], w["sampler"])
                pos = next(it)
                corrupt = smp.sample(pos, 1, seed=g)
                if ktup:
                    m.kg_loss_step_corrupt(pos, corrupt, margin=1.0)
                else:
                    m.loss_step_corrupt(pos, corrupt, margin=1.0)
            torch.nn.utils.clip_grad_norm_(params, 5.0, foreach=True)
            opt.step()
    return run


def timed_us(run, steps):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    run(steps)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / steps


def leg_steps(names, steps, rounds):
    runners = {}
    for name in names:
        for mode in ("touched", "all"):
            runners[(name, mode)] = graph_runner(make(name, mode))
        runners[(name, "torch_dense")] = dense_runner(make(name, "touched"))
    for r in runners.values():             # warm-up: captures, allocator, clocks
        r(steps)
    res = {}
    for _ in range(rounds):                # alternated in one session
        for key, r in runners.items():
            res.setdefault(key, []).append(timed_us(r, steps))
    out = {}
    for name in names:
        d = {mode: {"us_per_step": res[(name, mode)]} for mode in ("touched", "all", "torch_dense")}
        d["all_over_touched"] = min(res[(name, "all")]) / min(res[(name, "touched")])
        d["torch_dense_over_all"] = min(res[(name, "torch_dense")]) / min(res[(name, "all")])
        out[name] = d
    return out


def _sweep_bytes(opt, tables, w):
    """Algorithmic bytes of one ALL sweep over `tables` with the current marks (epoch opt.t)."""
    n_state = sum(x is not None for x in (opt.s1[tables[0]], opt.s2[tables[0]]))
    total = 0
    for k in tables:
        rows, dim = w[k].shape
        total += rows * dim * 4 * 2 * (1 + n_state)               # p and the rule's state, read and written
        mk = opt.marks.get(k)
        if mk is not None:
            marked = int((mk == opt.t).sum())
            total += marked * dim * 4 * 2 + rows * 4               # acc read + cleared, the marks
        else:
            total += rows * dim * 4 * 2                            # every row is marked
    return total


def leg_sweep(names, iters):
    import ctypes as C
    from torch.profiler import ProfilerActivity, profile
    from kgrec_b200 import _lib
    from kgrec_b200 import functional as KF
    out = {}
    for name in names:
        w = make(name, "all")
        opt = w["opt"]
        graph_runner(w)(10)                 # one step of each kind: marks of the last one stay (epoch opt.t)
        torch.cuda.synchronize()
        weights = w["model"]._weights()
        calls = {"all": opt.names} if name != "ktup_adam" else {"rec": opt.names, "kg": ("ent", "rel", "norm")}
        for call, tables in calls.items():
            ents = [_lib.OptTable(table=weights[k].data_ptr(), acc=opt.acc[k].data_ptr(),
                                  state1=opt.s1[k].data_ptr() if opt.s1[k] is not None else None,
                                  state2=opt.s2[k].data_ptr() if opt.s2[k] is not None else None,
                                  marks=opt.marks[k].data_ptr() if k in opt.marks else None,
                                  rows=weights[k].shape[0], dim=weights[k].shape[1], keep_acc=0) for k in tables]
            arr = (_lib.OptTable * len(ents))(*ents)
            i0 = opt.names.index(tables[0])
            kind, lr, wd = WORK[name]
            P = _lib.OptParams(kind=opt.kind, rows=_lib.ROWS_ALL, lr=lr, eps=opt.eps, beta1=0.9, beta2=0.999, alpha=0.99,
                               momentum=0.0, weight_decay=wd, max_norm=5.0,
                               step_counts=(opt.steps.data_ptr() + 8 * i0) if opt.steps is not None else None)
            nbytes = _sweep_bytes(opt, tables, weights)
            lib = _lib.load()

            def call_once():
                _lib.check(lib.kgrec_rows_update_ex(arr, len(ents), opt.t, C.byref(P), KF._ptr(opt.sqnorm), KF._stream()))
            for _ in range(5):
                call_once()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(iters):
                    call_once()
                torch.cuda.synchronize()
            times = [e.time_range.elapsed_us() for e in prof.events()           # the kernels' own intervals, us
                     if "k_rows_update_all" in e.name and e.device_type == torch.autograd.DeviceType.CUDA]
            times.sort()
            med = times[len(times) // 2]
            out["%s/%s" % (name, call)] = {"kernels": len(times), "median_us": med, "min_us": times[0],
                                           "algorithmic_MB": nbytes / 1e6, "GBps": nbytes / (med * 1e-6) / 1e9,
                                           "fraction_of_3.35TBps": nbytes / (med * 1e-6) / PEAK}
        del w
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--leg", choices=("steps", "sweep"), default="steps")
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--workloads", default=",".join(WORK))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("optimizer_rows.py needs a GPU")
    names = a.workloads.split(",")
    info = gpu_info()
    out = {"leg": a.leg, "batch_size": BATCH, "d": D}
    if a.leg == "steps":
        out.update(steps=a.steps, rounds=a.rounds, results=leg_steps(names, a.steps, a.rounds))
    else:
        out.update(iters=a.iters, results=leg_sweep(names, a.iters))
    out["gpu"] = info
    out["gpu_after"] = gpu_info()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
