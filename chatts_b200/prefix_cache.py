"""Prefix caching: the KV pages of a prompt prefix that an earlier prefill already wrote are reused instead of recomputed.

A ChatTS prompt is mostly time series, and the common workloads resend the same series (several questions about one set of series,
every turn of a chat that resends its history, ``n > 1`` completions).  A cache keyed on token ids alone would see every ``<ts>``
placeholder as the same token, so the key of a page covers what the model actually computes at its positions:

  * the key of full page k of a sequence's MERGED layout is h_k = H(h_{k-1}, contents of page k), a chain, so a page is shared only
    when everything in front of it is shared too;
  * the contents of a text position are its token id; of a patch-row position, a digest of that series' bytes as passed to the model
    plus the patch index;
  * the chain starts from a seed that covers the merge mode, the page size and a weights epoch, which every weight change bumps.

Two prompts with identical token ids and different series therefore share no page from the first ``<ts>`` page on.  Only full pages
of prompt positions are indexed, and a hit stops one position short of the prompt's end, so the last prompt position (whose logits
are needed) is always recomputed and every decode write lands in a private page.
"""
import hashlib
from collections import OrderedDict

import numpy as np
import torch


def _h(*parts):
    m = hashlib.blake2b(digest_size=16)
    for p in parts:
        m.update(p)
    return m.digest()


def chain_seed(mode, page_size, epoch):
    return _h(f"chatts-prefix-cache/merge={mode}/page={int(page_size)}/epoch={int(epoch)}".encode())


def series_digests(timeseries):
    """16-byte digest per series of ``timeseries`` [N, ...]: its dtype and values up to the last non-zero element (the zero padding a
    batch adds to its shorter series does not change what the encoder computes, so it does not change the key either)."""
    if timeseries is None or timeseries.shape[0] == 0:
        return []
    x = timeseries.detach().reshape(timeseries.shape[0], -1).cpu().contiguous()
    out = []
    for i in range(x.shape[0]):
        row = x[i]
        nz = torch.nonzero(row)
        row = row[: int(nz[-1, 0]) + 1 if nz.shape[0] else 0].contiguous()
        out.append(_h(str(row.dtype).encode(), row.view(torch.uint8).numpy().tobytes()))
    return out


def page_keys(lay, digests, patch_cnt, seed, page_size):
    """Chained keys of the full pages of every sequence of the merged layout ``lay`` (layout.MergedLayout): a list per sequence."""
    T = lay.total
    content = np.zeros((T, 3), dtype=np.uint64)             # text: (0, id, 0); patch row r of a series: (1 + r, digest)
    text = lay.ids >= 0
    content[text, 1] = lay.ids[text].astype(np.uint64)
    cnt = np.asarray(patch_cnt, dtype=np.int64).reshape(-1)
    if lay.row_map.shape[0] > 0:
        series = np.repeat(np.arange(cnt.shape[0]), cnt)
        within = np.arange(series.shape[0]) - (np.cumsum(cnt) - cnt)[series]
        dig = np.frombuffer(b"".join(digests), dtype=np.uint64).reshape(-1, 2) if digests else np.zeros((0, 2), np.uint64)
        content[lay.row_map, 0] = (1 + within).astype(np.uint64)
        content[lay.row_map, 1:] = dig[series]
    keys = []
    cu = lay.cu_seqlens
    for b in range(cu.shape[0] - 1):
        h, ks = seed, []
        for k in range((int(cu[b + 1]) - int(cu[b])) // page_size):
            a = int(cu[b]) + k * page_size
            h = _h(h, content[a:a + page_size].tobytes())
            ks.append(h)
        keys.append(ks)
    return keys


class CachingPagePool:
    """The page allocator of a model with prefix caching on: PagePool's free list plus reference counts and an index of the pages
    that hold a full page of some prompt (key -> page).

      * a cached page whose count drops to 0 becomes evictable, not free: a later prompt can still hit it;
      * alloc takes never-cached free pages first, then evicts the least recently released cached pages;
      * release takes a sequence's pages in page-table order and drops them deepest first, so the tail of a chain is evicted before
        its head (a head without its tail still serves hits, a tail without its head never does)."""

    def __init__(self, num_pages):
        self.free = list(range(num_pages - 1, -1, -1))
        self.num_pages = num_pages
        self.ref = {}                                        # page -> reference count, for every page in use or in the index
        self.page_of, self.key_of = {}, {}                   # key <-> page of the indexed pages
        self.evictable = OrderedDict()                       # indexed pages with count 0, least recently released first
        self.evictions = 0

    def available(self):
        return len(self.free) + len(self.evictable)

    def lookup(self, keys):
        """Pages of the longest run of ``keys`` (a chain) that is in the index."""
        pages = []
        for k in keys:
            p = self.page_of.get(k)
            if p is None:
                break
            pages.append(p)
        return pages

    def acquire(self, pages):
        for p in pages:
            self.evictable.pop(p, None)
            self.ref[p] = self.ref.get(p, 0) + 1

    def alloc(self, n):
        if n > self.available():
            raise RuntimeError(f"KV cache exhausted: need {n} pages, {self.available()} free or evictable of {self.num_pages}")
        out = []
        for _ in range(n):
            if self.free:
                p = self.free.pop()
            else:
                p, _ = self.evictable.popitem(last=False)
                del self.page_of[self.key_of.pop(p)]
                del self.ref[p]
                self.evictions += 1
            self.ref[p] = 1
            out.append(p)
        return out

    def release(self, pages):
        for p in reversed(pages):
            n = self.ref[p] - 1
            if n > 0:
                self.ref[p] = n
            elif p in self.key_of:
                self.ref[p] = 0
                self.evictable[p] = None
            else:
                del self.ref[p]
                self.free.append(p)

    def register(self, key, page):
        """Index ``page`` (in use, its contents final) under ``key``; a key or page already in the index is left as it is."""
        if key in self.page_of or page in self.key_of:
            return False
        self.page_of[key] = page
        self.key_of[page] = key
        return True

    def clear(self):
        """Drops the whole index: evictable pages become free, pages in use become private pages of their holders."""
        for p in self.evictable:
            del self.ref[p]
            self.free.append(p)
        self.evictable.clear()
        self.page_of.clear()
        self.key_of.clear()
