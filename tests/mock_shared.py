"""TEST INFRASTRUCTURE: the mock kernel layer for request-queue calls that share prompts, on top of tests/mock_rows.py.

A shared prompt is prefilled at batch 1 through one row of the block table over the whole pools, so the row's page ids
run past the batch-1 range that tests/mock_kernels.py's `_pool` views.  Here `_pool` views every pool a PagedKV
allocated at its full size; any other pointer keeps the batch * max_pages view.
"""
import mock_kernels as MK
import mock_rows

POOLS = {}                  # data_ptr of a PagedKV pool -> its page count


def install(monkeypatch, persist=False):
    """mock_rows.install plus full-size pool views, for the duration of one test."""
    from midi_b200 import decode
    mock_rows.install(monkeypatch, persist=persist)
    POOLS.clear()
    init, pool = decode.PagedKV.__init__, MK._pool

    def paged_init(self, *a, **k):
        init(self, *a, **k)
        for t in self.k + self.v:
            POOLS[t.data_ptr()] = t.shape[0]

    def full_pool(ptr, batch, max_pages, nh, page, D):
        n = POOLS.get(ptr)
        return pool(ptr, batch, max_pages, nh, page, D) if n is None else pool(ptr, 1, n, nh, page, D)

    monkeypatch.setattr(decode.PagedKV, "__init__", paged_init)
    monkeypatch.setattr(MK, "_pool", full_pool)
