"""Helpers of the PatchCleanser sharding tests (not a test module).

ThreadWorld runs `world` ranks as threads of one process: each thread gets a rank object with the part of the
torch.distributed API the sharding helpers use (get_rank, get_world_size, get_backend, all_gather), and all_gather
meets the other threads at a barrier.  On a GPU the ranks share one engine, so their forwards run in turn under a lock:
a simulated world on one device, where each rank's share is forwarded exactly as a real rank would forward it.

FakeEngine stands in for the engine on the CPU: the label of every sample is looked up in a scenario (round-1 sample j,
second-round sample (j, k), certificate sample d), decoded from its rectangles or mask-bank indices, and the samples of
every chunk it would run are recorded."""
import threading

import numpy as np
import torch

from dorpatch_b200 import masks as PM


class _Rank:
    def __init__(self, world, rank):
        self._w, self._r = world, rank

    def get_rank(self):
        return self._r

    def get_world_size(self):
        return self._w.world

    def get_backend(self):
        return "gloo"

    def all_gather(self, outs, t):
        w = self._w
        w.slots[self._r] = t.detach().cpu().clone()
        w.barrier.wait()
        for o, s in zip(outs, w.slots):
            o.copy_(s)
        w.barrier.wait()


class ThreadWorld:
    def __init__(self, world):
        self.world = world
        self.barrier = threading.Barrier(world, timeout=600)
        self.slots = [None] * world

    def run(self, fn):
        """[fn(rank object) for every rank], each on its own thread; re-raises the first failure."""
        out, err = [None] * self.world, [None] * self.world

        def body(r):
            try:
                out[r] = fn(_Rank(self, r))
            except BaseException as ex:           # a failed rank breaks the barrier, so no other rank waits forever
                err[r] = ex
                self.barrier.abort()

        ts = [threading.Thread(target=body, args=(r,)) for r in range(self.world)]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        for e in err:
            if e is not None and not isinstance(e, threading.BrokenBarrierError):
                raise e
        for e in err:
            if e is not None:
                raise e
        return out


class FakeEngine:
    """Labels by scenario: round-1 sample j -> first[j]; second-round sample (j, k) -> second(j, k); certificate sample
    d -> cert[d].  Samples are decoded from the window's rectangle tables (mw) or, on a mask bank, from the indices
    (the bank of n_single masks is the singles' one).  `chunks` lists, per chunk the engine would run, its samples."""

    def __init__(self, chunk, mw, first, second, cert):
        self.chunk, self.first, self.second, self.cert = chunk, np.asarray(first), second, np.asarray(cert)
        single = PM.gather(mw.mask_rects, np.arange(len(mw.mask_rects)))
        double = PM.gather(mw.double_mask_rects, np.arange(len(mw.double_mask_rects)))
        self.n_single = len(single)
        self._single = {r.tobytes(): j for j, r in enumerate(single)}
        self._double = {r.tobytes(): d for d, r in enumerate(double)}
        self.chunks = []

    def _decode(self, row):
        d = self._double.get(row.tobytes())
        if d is not None:
            return ("c", int(d), -1)
        head = row.copy()
        head[2:4] = 0
        j = self._single[head.tobytes()]
        if not row[2:4].any():
            return ("1", int(j), -1)
        tail = np.zeros_like(row)
        tail[0:2] = row[2:4]
        return ("2", int(j), int(self._single[tail.tobytes()]))

    def _label(self, s):
        kind, a, b = s
        return int(self.first[a]) if kind == "1" else (int(self.second(a, b)) if kind == "2" else int(self.cert[a]))

    def predict(self, x, S, rects=None, bank=None, idx=None):
        if bank is not None:
            idx = np.asarray(idx).reshape(S, -1)
            k = idx[:, 1] if idx.shape[1] > 1 else np.full(S, -1)
            if bank.shape[0] == self.n_single:
                samples = [("1", int(j), -1) if kk < 0 else ("2", int(j), int(kk)) for j, kk in zip(idx[:, 0], k)]
            else:
                samples = [("c", int(d), -1) for d in idx[:, 0]]
        else:
            samples = [self._decode(r) for r in np.asarray(rects).reshape(S, 4, 4)]
        for c0 in range(0, S, self.chunk):
            self.chunks.append(tuple(samples[c0:c0 + self.chunk]))
        return np.array([self._label(s) for s in samples], np.int32)


def scenarios(n1, n2, majority=5):
    """(name, first, second, cert) covering: a unanimous image certified, a unanimous image with one certificate
    disagreement, and a second-round image with two confirmed minority labels (2 via sample 3, 8 via sample 7; the
    last confirmed in the iteration order must win), two failing checks (label 2 via sample 20, label 9 via the last
    sample, each failing on one second-round sample only) and one certificate disagreement."""
    out = []
    unanimous = np.full(n1, majority)
    cert = np.full(n2, majority)
    out.append(("unanimous", unanimous, lambda j, k: majority, cert))
    bad = cert.copy()
    bad[n2 - 1] = 3
    out.append(("unanimous_cert_fails", unanimous, lambda j, k: majority, bad))
    first = unanimous.copy()
    first[[3, 20]] = 2
    first[7] = 8
    first[n1 - 1] = 9
    confirm = {3, 7}

    def second(j, k):
        return first[k] if (k in confirm or j != n1 - 1) else majority
    bad2 = cert.copy()
    bad2[1] = 2
    out.append(("round2", first, second, bad2))
    return out


def records_equal(a, b):
    same = type(a.prediction) is type(b.prediction) and a.prediction == b.prediction \
        and type(a.certification) is type(b.certification) and a.certification == b.certification \
        and a.preds_1.dtype == b.preds_1.dtype and np.array_equal(a.preds_1, b.preds_1)
    if a.preds_2 is None or b.preds_2 is None:
        return same and a.preds_2 is None and b.preds_2 is None
    return same and a.preds_2.dtype == b.preds_2.dtype and np.array_equal(a.preds_2, b.preds_2)


def expected_prediction(first, second):
    """The reference's prediction (PatchCleanser.py:74-90) for a scenario, worked out from the scenario alone: the
    majority of round 1, unless some minority sample k has every second-round sample (j, k) labelled like k; then the
    last such label in the reference's iteration order (labels as unique(sorted=False) gives them, k ascending).
    Returns (prediction, the set of confirmed labels)."""
    first = np.asarray(first, np.int64)
    labels, counts = torch.from_numpy(first).unique(sorted=False, return_counts=True)
    majority = labels[counts.argmax()].item()
    pred, confirmed = majority, set()
    if len(labels) > 1:
        n = len(first)
        for label in labels.tolist():
            if label == majority:
                continue
            for k in np.nonzero(first == label)[0]:
                if all(second(j, k) == label for j in range(n)):
                    pred = label
                    confirmed.add(label)
    return pred, confirmed
