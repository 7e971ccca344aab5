"""The NN-worker side forward engine: prefetch, ordering, bounded staleness (SURVEY.md N1).

Mirrors rust/persia-core/src/forward.rs:
  * `PerisaDataOrderManager` (:396-468): with `reproducible`, batches are released in batch-id order — the next
    expected id starts at the replica's rank and advances by the world size; when nothing arrives for a second the
    buffered batches are flushed in id order (the reference logs a warning and does the same);
  * `ForwardImpl` (:470-780): `num_workers` lookup workers take batches off the (re-ordered) input, look their
    embeddings up and queue the result, at most `forward_buffer_size` deep; a batch whose ids were sent ahead to the
    embedding worker (`IDTypeFeatureRemoteRef`) first takes one of `embedding_staleness` permits (:687-690), which
    travels with the training batch into its gradient batch and is returned when the update has been applied
    (backward.rs:286-343) — so at most that many batches are between lookup and update;
  * `get_batch(timeout_ms)` raises TimeoutError (:875).

Host-side threads only: the lookup itself is a callable (persia_core passes the pb_forward path), so this module
never touches the GPU and is tested on the CPU with a stand-in lookup.
"""
import heapq
import itertools
import logging
import queue
import threading
import time

_log = logging.getLogger(__name__)


class Permit:
    """One unit of embedding staleness; returning it twice is harmless (OwnedSemaphorePermit is dropped once)."""

    def __init__(self, sem):
        self._sem = sem

    def release(self):
        sem, self._sem = self._sem, None
        if sem is not None:
            sem.release()

    def __del__(self):
        self.release()


class ForwardEngine:
    def __init__(self, lookup, forward_buffer_size, reproducible, embedding_staleness=None, world_size=1, rank=0,
                 flush_after_s=1.0, stage=None):
        """lookup(batch, permit_or_None) -> training batch.  `is_remote_ref(batch)` decides who needs a permit.
        stage(batch), optional: called by the worker on every batch it takes in, before it waits for the batch's
        permit, so that work which needs only the batch's ids (persia_core: the host-tier moves of its lookup) runs
        while the batches before it still train.  An error is logged and the batch goes on: the lookup does the same
        work anyway."""
        self.lookup = lookup
        self.stage = stage
        self.reproducible = bool(reproducible)
        self.world_size, self.rank, self.flush_after_s = max(1, int(world_size)), int(rank), float(flush_after_s)
        self._out = queue.Queue(maxsize=max(1, int(forward_buffer_size)))
        self._ordered = queue.Queue(maxsize=1) if self.reproducible else None  # flume::bounded(1), forward.rs:498
        self._sem = threading.Semaphore(int(embedding_staleness)) if embedding_staleness else None
        self._input = None
        self._running = threading.Event()
        self._threads = []
        self.is_remote_ref = lambda batch: False

    # ---- wiring ---------------------------------------------------------------------------------------
    def set_input(self, q):
        if self._input is not None:
            raise RuntimeError("do not set input channel again")
        self._input = q

    def launch(self, num_workers):
        if self._threads:
            return  # "forward engine already launch"
        if self._input is None:
            raise RuntimeError("please set input channel before launch the forward engine")
        self._running.set()
        if self.reproducible:
            self._spawn(self._reorder_loop, "persia-forward-reorder")
        for i in range(max(1, int(num_workers))):
            self._spawn(self._worker_loop, f"persia-forward-{i}")

    def shutdown(self):
        self._running.clear()
        for t in self._threads:
            t.join(timeout=2.0)
        self._threads = []

    def get_batch(self, timeout_ms):
        if not self._threads:
            raise RuntimeError("forward engine is not launched")
        try:
            item = self._out.get(timeout=max(int(timeout_ms), 1) / 1000.0)
        except queue.Empty:
            raise TimeoutError("get train batch timed out")
        if isinstance(item, BaseException):
            raise item
        return item

    # ---- threads --------------------------------------------------------------------------------------
    def _spawn(self, fn, name):
        t = threading.Thread(target=fn, name=name, daemon=True)
        t.start()
        self._threads.append(t)

    def _put(self, q, item):
        while self._running.is_set():
            try:
                q.put(item, timeout=0.01)
                return True
            except queue.Full:
                continue
        return False

    def _reorder_loop(self):
        heap, tie = [], itertools.count()
        expect, last_pop = self.rank, time.monotonic()

        def pop():
            nonlocal expect, last_pop
            _, _, bid, batch = heapq.heappop(heap)
            last_pop = time.monotonic()
            expect = (bid if bid is not None else expect) + self.world_size
            return batch

        while self._running.is_set():
            try:
                batch = self._input.get(timeout=0.01)
            except queue.Empty:
                if heap and time.monotonic() - last_pop > self.flush_after_s:  # the input is slow: stop waiting
                    while heap and self._put(self._ordered, pop()):
                        pass
                continue
            bid = getattr(batch, "_batch_id", None)
            heapq.heappush(heap, (bid if bid is not None else -1, next(tie), bid, batch))  # None sorts first (usize::MIN)
            while heap and heap[0][0] <= expect:
                if not self._put(self._ordered, pop()):
                    return

    def _worker_loop(self):
        src = self._ordered if self.reproducible else self._input
        while self._running.is_set():
            try:
                batch = src.get(timeout=0.01)
            except queue.Empty:
                continue
            if self.stage is not None:
                try:
                    self.stage(batch)
                except Exception:  # noqa: BLE001 — the lookup restores what the stage did not move
                    _log.exception("staging a batch failed; its lookup moves its entries itself")
            permit = None
            if self._sem is not None and self.is_remote_ref(batch):
                while not self._sem.acquire(timeout=0.01):
                    if not self._running.is_set():
                        return
                permit = Permit(self._sem)
            try:
                item = self.lookup(batch, permit)
            except BaseException as e:  # noqa: BLE001 — surfaced to the consumer by get_batch
                if permit is not None:
                    permit.release()
                item = e
            if not self._put(self._out, item) and permit is not None:
                permit.release()
