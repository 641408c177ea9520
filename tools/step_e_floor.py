#!/usr/bin/env python
"""How far the TransE step kernel is from the memory traffic it cannot avoid.

    python tools/step_e_floor.py [--entities 100000,500000,5000000] [--min-seconds 0.5]

Prints ONE JSON line with, for each table size, the mean time per launch of

  step    kgrec_corrupt_loss_step through the module API (TransEModel.loss_step_corrupt, sparse slot
          gradients) on bench.py's workload: d=100, 256 batches of 1024 positives x 10 corrupted negatives,
          the bench's table and id seeds, three index sets in rotation;
  gather  torch.index_select of the same (2 + K) entity rows and one relation row per group into slot
          buffers of the step's shape: the step's row reads and slot writes with no arithmetic;
  write   zero_() over as many bytes as the step writes (slot rows, slot ids, scores, group losses);

and the DRAM-side rate of each from byte counts computed from the shapes.  The card name, power limit and
SM clock are read in the same call.  CUDA events, warm-up, and at least --min-seconds of timed work per figure.
There is no CPU fallback: without a GPU the script fails.
"""
import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "joint-kg-recommender_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

from bench import BATCH, D, K_NEG, N_REL, make_indices  # noqa: E402

N_BATCHES = 256                 # bench.py --batches-per-step


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        return dict(zip(q.split(","), (c.strip() for c in out.strip().split(","))))
    except Exception as e:            # the timing does not depend on it; say why it is missing
        return {"name": torch.cuda.get_device_name(), "error": repr(e)}


def time_per_call(fn, min_seconds):
    """Mean ms per call over at least min_seconds of back-to-back calls, after a warm-up."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(5):
        fn()
    b.record()
    torch.cuda.synchronize()
    reps = max(10, math.ceil(min_seconds * 1e3 / (a.elapsed_time(b) / 5)))
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps, reps


def measure(K, n_ent, min_seconds, dev):
    from kgrec_b200.models.base import device_init
    torch.manual_seed(0)
    if n_ent == 100_000:              # bench.py's headline model and ids
        model = K.TransEModel(False, D, n_ent, N_REL)
        gen = torch.Generator().manual_seed(1234)
    else:                             # bench.py's roofline.hbm_regime models and ids
        with device_init(dev):
            model = K.TransEModel(False, D, n_ent, N_REL)
        gen = torch.Generator().manual_seed(77)
    model.grad_mode = "sparse"
    sets = [[x.to(dev) for x in make_indices(torch, gen, N_BATCHES, n_ent=n_ent)] for _ in range(3)]
    n_pos = N_BATCHES * BATCH
    cnt = [0]

    def step():
        ix = sets[cnt[0] % 3]
        cnt[0] += 1
        model.zero_grad(set_to_none=True)
        model.loss_step_corrupt(tuple(ix[:3]), ix[3], margin=1.0, batch_pos=BATCH)

    step_ms, step_reps = time_per_call(step, min_seconds)

    # the slot row ids of each index set, as the step writes them
    ent_w, rel_w = model.ent_embeddings.weight.detach(), model.rel_embeddings.weight.detach()
    slot_sets = []
    for ix in sets:
        model.zero_grad(set_to_none=True)
        model.loss_step_corrupt(tuple(ix[:3]), ix[3], margin=1.0, batch_pos=BATCH)
        slot_sets.append((model.ent_embeddings.weight.grad._indices()[0].clone(),
                          model.rel_embeddings.weight.grad._indices()[0].clone()))
    model.zero_grad(set_to_none=True)
    ent_buf = torch.empty((n_pos * (2 + K_NEG), D), dtype=torch.float32, device=dev)
    rel_buf = torch.empty((n_pos, D), dtype=torch.float32, device=dev)

    def gather():
        se, sr = slot_sets[cnt[0] % 3]
        cnt[0] += 1
        torch.index_select(ent_w, 0, se, out=ent_buf)
        torch.index_select(rel_w, 0, sr, out=rel_buf)

    gather_ms, gather_reps = time_per_call(gather, min_seconds)
    del ent_buf, rel_buf, slot_sets

    row = 4 * D
    slot_rows = n_pos * (2 + K_NEG) + n_pos
    b_slots = slot_rows * row                                             # gradient slot rows written
    b_small = slot_rows * 8 + n_pos * 4 + n_pos * K_NEG * 4 + n_pos * 4   # slot ids, scores, group losses
    b_gather = slot_rows * row                                            # rows gathered (L2 or DRAM)
    b_ids = n_pos * 3 * 4 + n_pos * K_NEG * 4                             # int32 ids read
    step_writes = b_slots + b_small
    zbuf = torch.empty(step_writes // 4, dtype=torch.float32, device=dev)
    write_ms, write_reps = time_per_call(zbuf.zero_, min_seconds)
    del zbuf

    def rates(ms, nbytes):
        return nbytes / (ms * 1e-3) / 1e9
    res = {
        "entities": n_ent, "table_MB": n_ent * row / 1e6,
        "step_ms": step_ms, "step_reps": step_reps,
        "gather_ms": gather_ms, "gather_reps": gather_reps,
        "write_ms": write_ms, "write_reps": write_reps,
        "step_over_gather": step_ms / gather_ms, "step_over_write": step_ms / write_ms,
        # DRAM-side rates: writes always reach DRAM; row reads do so once the table does not fit L2
        "step_write_GBs": rates(step_ms, step_writes),
        "step_all_GBs": rates(step_ms, step_writes + b_gather + b_ids),
        "gather_write_GBs": rates(gather_ms, b_slots),
        "gather_all_GBs": rates(gather_ms, b_slots + b_gather + slot_rows * 8),
        "write_GBs": rates(write_ms, step_writes),
        "triples_per_s": n_pos * (1 + K_NEG) / (step_ms * 1e-3),
    }
    del model, sets
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--entities", default="100000,500000,5000000")
    ap.add_argument("--min-seconds", type=float, default=0.5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("step_e_floor.py measures on a GPU; none is visible")
    import kgrec_b200 as K
    dev = torch.device("cuda", torch.cuda.current_device())
    info_before = gpu_info()
    sizes = [measure(K, int(n), args.min_seconds, dev) for n in args.entities.split(",")]
    out = {"gpu": info_before, "gpu_after": gpu_info(), "shape": {"d": D, "batches": N_BATCHES, "batch": BATCH, "k_neg": K_NEG},
           "sizes": sizes}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
