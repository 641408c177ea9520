"""Host -> device staging of index batches.

The reference builds every batch as Python lists and uploads six LongTensors synchronously
per step (knowledge_representation.py:179-184).  DevicePrefetcher keeps that contract -- the
caller hands over host (ideally pinned) index tensors, the model gets device tensors -- but
issues the copies of batch i+1 on a side stream while batch i is being scored, into a fixed
ring of device staging buffers (no allocation in steady state: an allocator round trip inside
the loop shows up as a multi-millisecond hiccup every few hundred launches).
"""
import torch


class DevicePrefetcher:
    """Iterate over host batches (tuples / lists of tensors), yielding device copies; the copy
    of the next batch overlaps the consumer's kernels.  Every tensor of a batch is copied inside
    the iteration that precedes its use, so a timed region around the loop contains all copies.
    The yielded tensors are views of a staging ring: they are valid until `depth` further batches
    have been requested (the consumer's kernels on them are ordered before the slot is reused)."""

    _streams = {}     # one copy stream per device for the life of the process
    _rings = {}       # staging rings keyed by (device, depth, shapes / dtypes): reused across epochs

    def __init__(self, batches, device, depth=2):
        self.it = iter(batches)
        self.device = torch.device(device)
        key = (self.device.type, self.device.index if self.device.index is not None else torch.cuda.current_device())
        if key not in DevicePrefetcher._streams:
            DevicePrefetcher._streams[key] = torch.cuda.Stream(device=self.device)
        self.copy_stream = DevicePrefetcher._streams[key]
        self.key = key
        self.queue = []
        self.depth = max(1, depth)
        self.slot = 0
        self.ring = None

    def _fresh(self, host):
        """New staging buffers.  The caching allocator may hand out memory whose previous owner's kernels are still
        queued on the CURRENT stream; the copy stream writes these buffers, so it must first catch up with it."""
        bufs = [torch.empty(x.shape, dtype=x.dtype, device=self.device) for x in host]
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.device))
        self.copy_stream.wait_event(ev)
        return bufs

    def _ring_for(self, host):
        sig = (self.key, self.depth, tuple((tuple(x.shape), x.dtype) for x in host))
        ring = DevicePrefetcher._rings.get(sig)
        if ring is None:
            n = self.depth + 1
            ring = {"bufs": [self._fresh(host) for _ in range(n)], "done": [None] * n}
            if len(DevicePrefetcher._rings) > 8:
                DevicePrefetcher._rings.clear()
            DevicePrefetcher._rings[sig] = ring
        return ring

    def _enqueue(self):
        try:
            host = next(self.it)
        except StopIteration:
            return False
        if self.ring is None:
            self.ring = self._ring_for(host)
        s = self.slot
        self.slot = (s + 1) % len(self.ring["bufs"])
        bufs = self.ring["bufs"][s]
        if len(bufs) != len(host) or any(b.shape != x.shape or b.dtype != x.dtype for b, x in zip(bufs, host)):
            bufs = self._fresh(host)                                                           # ragged last batch
            self.ring["done"][s] = None
        with torch.cuda.stream(self.copy_stream):
            if self.ring["done"][s] is not None:
                self.copy_stream.wait_event(self.ring["done"][s])      # the consumer's kernels on this slot are done
            for b, x in zip(bufs, host):
                b.copy_(x, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self.copy_stream)
        self.queue.append((bufs, ev, host, s))
        return True

    def __iter__(self):
        while len(self.queue) < self.depth and self._enqueue():
            pass
        while self.queue:
            dev, ev, _host, s = self.queue.pop(0)
            cur = torch.cuda.current_stream(self.device)
            cur.wait_event(ev)
            self._enqueue()
            yield dev
            done = torch.cuda.Event()          # the consumer has enqueued its work on this batch by now
            done.record(torch.cuda.current_stream(self.device))
            self.ring["done"][s] = done


class DeviceTrainIterator:
    """The reference's endless training iterator (``MakeTrainIterator``, utils/data.py:87-110) with the training set
    resident on the device: no Python lists, no per-step host -> device copies.

    Same epoch rule as the reference, including its quirk: the visiting order is ``range(n)`` repeated
    ``negtive_samples`` times and shuffled, a batch is ``order[start : start + batch_size]``, and a new epoch (a fresh
    shuffle, ``start = 0``) begins as soon as ``start > n - batch_size`` -- so an epoch yields
    ``(n - batch_size) // batch_size + 1`` batches drawn from the first ``n`` entries of the shuffled order whatever
    ``negtive_samples`` is.  The shuffle is ``torch.randperm`` on the data's device from a private generator
    (reproducible per seed; not the reference's ``random.shuffle`` stream).

    data: [n, c] integer tensor or array (triples ``h, t, r`` / ratings ``u, i``).  Yields a tuple of ``c`` contiguous
    device index tensors of ``batch_size`` entries -- what ``SparseRowOptimizer.step_corrupt`` / ``step_pairs`` and the
    negative samplers (kgrec_b200.sampling) consume."""

    def __init__(self, data, batch_size, negtive_samples=1, device="cuda", seed=0, dtype=torch.int32):
        rows = torch.as_tensor(data)
        if rows.dim() != 2 or rows.shape[0] == 0:
            raise ValueError("DeviceTrainIterator: data must be a non-empty [n, columns] integer array")
        if batch_size < 1 or negtive_samples < 1:
            raise ValueError("DeviceTrainIterator: batch_size and negtive_samples must be >= 1")
        self.device = torch.device(device)
        self.cols = [rows[:, c].to(self.device, dtype).contiguous() for c in range(rows.shape[1])]   # column-major: one gather each
        self.n = rows.shape[0]
        self.batch_size = int(batch_size)
        self.repeat = int(negtive_samples)
        self.gen = torch.Generator(device=self.device)
        self.gen.manual_seed(int(seed))
        self.epoch = 0
        self.start = -self.batch_size
        self._shuffle()

    def _shuffle(self):
        # list(range(n)) * k shuffled == a random permutation of the multiset: permute k*n slots, fold by n
        perm = torch.randperm(self.n * self.repeat, generator=self.gen, device=self.device)
        self.order = perm % self.n if self.repeat > 1 else perm

    @property
    def batches_per_epoch(self):
        return max(0, (self.n - self.batch_size)) // self.batch_size + 1

    def batches_left(self):
        """Batches __next__ yields before it starts a new epoch (host arithmetic only, nothing is read back)."""
        return max(0, (self.n - self.batch_size - self.start) // self.batch_size)

    def __iter__(self):
        return self

    def __next__(self):
        self.start += self.batch_size
        if self.start > self.n - self.batch_size:
            self.start = 0
            self.epoch += 1
            self._shuffle()
        idx = self.order[self.start:self.start + self.batch_size]
        return tuple(c.index_select(0, idx) for c in self.cols)
