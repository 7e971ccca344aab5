"""CPU: ForwardEngine's stage hook (persia_b200/engine.py) — called once per batch, in arrival order, before the batch
waits for its staleness permit, so that a batch's host-tier moves overlap the batches still training before it; a
failing stage loses no batch.  A stand-in lookup and stage record what happens."""
import queue
import threading
import time

from persia_b200.engine import ForwardEngine


class B:
    def __init__(self, bid, ref=True):
        self._batch_id, self.ref = bid, ref


class LoggingSemaphore:
    """threading.Semaphore that notes every permit taken."""

    def __init__(self, n, log):
        self._s, self._log = threading.Semaphore(n), log

    def acquire(self, timeout=None):
        ok = self._s.acquire(timeout=timeout)
        if ok:
            self._log.append("permit")
        return ok

    def release(self):
        self._s.release()


def _engine(stage, staleness=None, buffer=8, log=None):
    q = queue.Queue()
    e = ForwardEngine(lambda b, p: (b._batch_id, p), buffer, False, staleness, stage=stage)
    if staleness and log is not None:
        e._sem = LoggingSemaphore(staleness, log)
    e.set_input(q)
    e.is_remote_ref = lambda b: b.ref
    return e, q


def test_stage_once_per_batch_in_arrival_order_before_the_permit():
    log = []
    e, q = _engine(lambda b: log.append(("stage", b._batch_id)), staleness=4, log=log)
    e.launch(1)
    try:
        for bid in range(6):
            q.put(B(bid))
        got = []
        for _ in range(6):
            bid, p = e.get_batch(2000)
            got.append(bid)
            p.release()
        assert got == list(range(6))
        assert [x for x in log if x != "permit"] == [("stage", i) for i in range(6)]
        assert log.count("permit") == 6
        for i in range(6):  # one worker: every batch's stage comes right before the permit it then waits for
            assert log[log.index(("stage", i)) + 1] == "permit", log
    finally:
        e.shutdown()


def test_stage_without_permits_and_without_a_stage():
    seen = []
    e, q = _engine(lambda b: seen.append(b._batch_id))
    e.launch(1)
    try:
        for bid in range(3):
            q.put(B(bid, ref=False))
        assert [e.get_batch(2000)[0] for _ in range(3)] == [0, 1, 2]
        assert seen == [0, 1, 2]
    finally:
        e.shutdown()
    e, q = _engine(None)
    e.launch(1)
    try:
        q.put(B(0, ref=False))
        assert e.get_batch(2000)[0] == 0
    finally:
        e.shutdown()


def test_raising_stage_loses_no_batch(caplog):
    def stage(b):
        if b._batch_id % 2:
            raise RuntimeError("stage failed")

    e, q = _engine(stage, staleness=2)
    e.launch(1)
    try:
        for bid in range(5):
            q.put(B(bid))
        got = []
        for _ in range(5):
            bid, p = e.get_batch(2000)
            got.append(bid)
            p.release()
        assert got == list(range(5))
    finally:
        e.shutdown()
    assert any("staging a batch failed" in r.getMessage() for r in caplog.records)


def test_next_stage_runs_while_the_previous_permit_is_held():
    """embedding_staleness 1: batch 1's stage runs while batch 0 still holds the one permit (its backward has not
    returned it), i.e. beside batch 0's training; batch 1's lookup waits for the permit."""
    log, staged = [], threading.Event()

    def stage(b):
        log.append(("stage", b._batch_id))
        if b._batch_id == 1:
            staged.set()

    e, q = _engine(stage, staleness=1, log=log)
    e.launch(1)
    try:
        q.put(B(0))
        q.put(B(1))
        bid, p0 = e.get_batch(2000)
        assert bid == 0
        assert staged.wait(2.0), log  # the permit of batch 0 is still held here
        time.sleep(0.05)
        assert log == [("stage", 0), "permit", ("stage", 1)], log
        try:
            e.get_batch(100)
            raise AssertionError("batch 1 was looked up without a permit")
        except TimeoutError:
            pass
        p0.release()
        bid, p1 = e.get_batch(2000)
        assert bid == 1 and log[-1] == "permit"
        p1.release()
    finally:
        e.shutdown()
