"""Device-resident ANS stream sets (host-side handle of `bsw_streams`).

One stream == one reference state list (cifar_compress.py:157-159): 32-bit
words bottom-first plus a 64-bit head.  `StreamSet` holds B of them in HBM."""
import ctypes

import numpy as np

from ._lib import lib, check, device_index, on_device


def _on_own_device(fn):
    import functools

    @functools.wraps(fn)
    def wrapper(self, *a, **k):
        with on_device(self.device):
            return fn(self, *a, **k)
    return wrapper


class StreamSet:
    def __init__(self, n_streams: int, capacity_words: int, device=None):
        self._h = ctypes.c_void_p()
        self.device = device_index(device)
        with on_device(self.device):
            check(lib().bsw_streams_create(ctypes.byref(self._h), int(n_streams), int(capacity_words)))
        self.n = int(n_streams)
        self.capacity = int(lib().bsw_streams_capacity(self._h))

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            try:
                lib().bsw_streams_destroy(h)
            except Exception:
                pass
            self._h = None

    @property
    def handle(self):
        return self._h

    # -- host <-> device --------------------------------------------------------------------
    @_on_own_device
    def fill(self, words, head):
        """Every stream := (words, head) -- the reference seeds each experiment identically."""
        w = np.ascontiguousarray(words, dtype=np.uint32)
        check(lib().bsw_streams_fill(self._h, w.ctypes.data, w.size, ctypes.c_uint64(int(head))))

    @_on_own_device
    def import_lists(self, states, first=0):
        """states: iterable of reference-style lists [w0, ..., w_{n-1}, head]."""
        states = list(states)
        offs = np.zeros(len(states) + 1, dtype=np.int64)
        for i, st in enumerate(states):
            offs[i + 1] = offs[i] + len(st) - 1
        words = np.zeros(max(int(offs[-1]), 1), dtype=np.uint32)
        heads = np.zeros(len(states), dtype=np.uint64)
        for i, st in enumerate(states):
            words[offs[i]:offs[i + 1]] = np.array(st[:-1], dtype=np.uint64).astype(np.uint32)
            heads[i] = st[-1]
        check(lib().bsw_streams_import(self._h, first, len(states), words.ctypes.data, offs.ctypes.data, heads.ctypes.data))

    @_on_own_device
    def import_packed(self, words, offsets, heads, first=0):
        """Inverse of export(): packed uint32 words + int64 offsets [count+1] + uint64 heads."""
        words = np.ascontiguousarray(words, dtype=np.uint32)
        offsets = np.ascontiguousarray(offsets, dtype=np.int64)
        heads = np.ascontiguousarray(heads, dtype=np.uint64)
        wp = words.ctypes.data if words.size else None
        check(lib().bsw_streams_import(self._h, first, len(heads), wp, offsets.ctypes.data, heads.ctypes.data))

    @_on_own_device
    def sizes(self):
        """(nwords int64[B], heads uint64[B], flags int32[B]) -- synchronises."""
        n = np.zeros(self.n, dtype=np.int64)
        h = np.zeros(self.n, dtype=np.uint64)
        f = np.zeros(self.n, dtype=np.int32)
        check(lib().bsw_streams_sizes(self._h, n.ctypes.data, h.ctypes.data, f.ctypes.data))
        return n, h, f

    @_on_own_device
    def min_words(self):
        """Lowest word count each stream reached since import/fill (reference: `excess_state_len - 1`)."""
        n = np.zeros(self.n, dtype=np.int64)
        check(lib().bsw_streams_min_words(self._h, n.ctypes.data))
        return n

    @_on_own_device
    def rest_words(self):
        """The reference's len(restbits) - 1 per stream (-1 until the chain reaches it): the word count after the first
        image's first pop for Bit-Swap (cifar_compress.py:190-192), after all its nz pops for BB-ANS (:224-226)."""
        n = np.zeros(self.n, dtype=np.int64)
        check(lib().bsw_streams_rest_words(self._h, n.ctypes.data))
        return n

    def bit_accounting(self, initial_words: int, xdim: int, images_per_chain: int):
        """The reference's per-chain bookkeeping (cifar_compress.py:253-259) from the current stream sizes:
        net = totaladdedbits / (xdim * images)  with totaladdedbits = (len(state) - len(initialstate)) * 32,
        cma = totalbits / (xdim * images)       with totalbits = (len(state) - (len(restbits) - 1)) * 32 -- the
        cumulative average INCLUDING the initial bits the first image's pops consumed up to restbits (rest_words)."""
        n, _, _ = self.sizes()
        rest = self.rest_words()
        added = (n - int(initial_words)) * 32.0
        total = (n + 1 - rest) * 32.0
        return dict(net_bits_per_dim=added / (xdim * images_per_chain), cma_bits_per_dim=total / (xdim * images_per_chain),
                    total_bits=total, total_added_bits=added)

    @_on_own_device
    def export(self, first=0, count=None):
        """Packed export: (words uint32[sum], offsets int64[count+1], heads uint64[count], flags)."""
        count = self.n - first if count is None else count
        n, h, f = self.sizes()
        n, h, f = n[first:first + count], h[first:first + count], f[first:first + count]
        offs = np.zeros(count + 1, dtype=np.int64)
        np.cumsum(n, out=offs[1:])
        words = np.zeros(max(int(offs[-1]), 1), dtype=np.uint32)
        check(lib().bsw_streams_export(self._h, first, count, words.ctypes.data, offs.ctypes.data))
        return words[:int(offs[-1])], offs, h, f

    # -- fast packed path: one gather/scatter kernel + three memcpys, pinned staging buffers -------------------------
    @_on_own_device
    def _staging(self, count, host=True):
        """Device staging buffers for `count` streams, and with host=True their pinned host twins (pack_device alone needs
        none: a worst-case pinned buffer of count * capacity words is costly to create)."""
        import torch
        st = getattr(self, "_stg", None)
        need = count * self.capacity
        if st is None or st["words_d"].numel() < need or st["offs_d"].numel() < count + 1:
            st = dict(words_d=torch.empty(need, dtype=torch.int32, device="cuda"),
                      offs_d=torch.empty(count + 1, dtype=torch.int64, device="cuda"),
                      heads_d=torch.empty(count, dtype=torch.int64, device="cuda"),
                      base_d=torch.empty(count, dtype=torch.int32, device="cuda"))
            self._stg = st
        if host and "words_h" not in st:
            n = st["offs_d"].numel() - 1
            st.update(base_h=torch.empty(n, dtype=torch.int32).pin_memory(),
                      words_h=torch.empty(st["words_d"].numel(), dtype=torch.int32).pin_memory(),
                      offs_h=torch.empty(n + 1, dtype=torch.int64).pin_memory(),
                      heads_h=torch.empty(n, dtype=torch.int64).pin_memory())
        return st

    @_on_own_device
    def pack_device(self, first=0, count=None, trim=False):
        """Device-side gather of the streams' words into one contiguous buffer, async on torch's current stream.
        Returns device tensors (words int32 [capacity view], offsets int64 [count+1], heads int64 [count],
        base int32 [count] or None).  trim=True packs only words[base_b .. n_b): the part above the lowest depth each
        stack ever reached (the untouched initial words below it are re-created by the receiver from the seed,
        demo_compress.py:137,160)."""
        from ._lib import cuda_stream_ptr
        count = self.n - first if count is None else count
        st = self._staging(count, host=False)
        if trim:
            check(lib().bsw_streams_pack_trimmed(self._h, first, count, st["words_d"].data_ptr(), st["offs_d"].data_ptr(),
                                                 st["heads_d"].data_ptr(), st["base_d"].data_ptr(), cuda_stream_ptr()))
        else:
            check(lib().bsw_streams_pack(self._h, first, count, st["words_d"].data_ptr(), st["offs_d"].data_ptr(),
                                         st["heads_d"].data_ptr(), cuda_stream_ptr()))
        return st["words_d"], st["offs_d"][:count + 1], st["heads_d"][:count], (st["base_d"][:count] if trim else None)

    @_on_own_device
    def unpack_device(self, words_d, offs_d, heads_d, base_d=None, first=0):
        """Inverse of pack_device from device tensors (e.g. what an NCCL gather delivered).  With base_d the streams must
        already hold their initial words (fill / import): the packed words are written above base_b."""
        from ._lib import cuda_stream_ptr
        count = heads_d.numel()
        if base_d is None:
            check(lib().bsw_streams_unpack(self._h, first, count, words_d.data_ptr(), offs_d.data_ptr(), heads_d.data_ptr(), cuda_stream_ptr()))
        else:
            check(lib().bsw_streams_unpack_trimmed(self._h, first, count, words_d.data_ptr(), offs_d.data_ptr(), heads_d.data_ptr(),
                                                   base_d.data_ptr(), cuda_stream_ptr()))

    @_on_own_device
    def export_packed(self, first=0, count=None, trim=False):
        """(words uint32[sum], offsets int64[count+1], heads uint64[count][, base int32[count]]) as numpy views of pinned
        host buffers (valid until the next export_packed/import_packed_fast).  Enqueued on torch's current stream;
        synchronises it.  trim=True: see pack_device."""
        import torch
        count = self.n - first if count is None else count
        st = self._staging(count)
        self.pack_device(first, count, trim)
        st["offs_h"][:count + 1].copy_(st["offs_d"][:count + 1], non_blocking=True)
        st["heads_h"][:count].copy_(st["heads_d"][:count], non_blocking=True)
        if trim:
            st["base_h"][:count].copy_(st["base_d"][:count], non_blocking=True)
        torch.cuda.current_stream().synchronize()
        total = int(st["offs_h"][count])
        st["words_h"][:total].copy_(st["words_d"][:total], non_blocking=True)
        torch.cuda.current_stream().synchronize()
        out = (st["words_h"][:total].numpy().view(np.uint32), st["offs_h"][:count + 1].numpy(),
               st["heads_h"][:count].numpy().view(np.uint64))
        return out + (st["base_h"][:count].numpy(),) if trim else out

    @_on_own_device
    def import_packed_fast(self, words, offsets, heads, first=0, base=None):
        """Inverse of export_packed (host arrays -> device scatter). Async on torch's current stream."""
        import torch
        count = len(heads)
        total = int(offsets[count])
        sent = np.diff(np.asarray(offsets[:count + 1], dtype=np.int64))
        if count and int(np.max(sent + (np.asarray(base[:count], dtype=np.int64) if base is not None else 0))) > self.capacity:
            raise OverflowError(f"import_packed_fast: a stream's base + packed length exceeds the capacity of {self.capacity} words")
        st = self._staging(count)
        if words.ctypes.data != st["words_h"].data_ptr():
            st["words_h"][:total].copy_(torch.from_numpy(np.ascontiguousarray(words).view(np.int32)))
            st["offs_h"][:count + 1].copy_(torch.from_numpy(np.ascontiguousarray(offsets, dtype=np.int64)))
            st["heads_h"][:count].copy_(torch.from_numpy(np.ascontiguousarray(heads).view(np.int64)))
            if base is not None:
                st["base_h"][:count].copy_(torch.from_numpy(np.ascontiguousarray(base, dtype=np.int32)))
        st["words_d"][:total].copy_(st["words_h"][:total], non_blocking=True)
        st["offs_d"][:count + 1].copy_(st["offs_h"][:count + 1], non_blocking=True)
        st["heads_d"][:count].copy_(st["heads_h"][:count], non_blocking=True)
        if base is not None:
            st["base_d"][:count].copy_(st["base_h"][:count], non_blocking=True)
        self.unpack_device(st["words_d"], st["offs_d"][:count + 1], st["heads_d"][:count],
                           st["base_d"][:count] if base is not None else None, first)

    def export_lists(self, first=0, count=None):
        words, offs, heads, flags = self.export(first, count)
        return [[int(v) for v in words[offs[i]:offs[i + 1]]] + [int(heads[i])] for i in range(len(heads))]

    def raise_on_error(self):
        """Maps per-stream status flags to the reference's exception types."""
        _, _, f = self.sizes()
        if (f == 1).any():
            raise IndexError(f"pop from empty ANS stack (streams {np.nonzero(f == 1)[0][:8].tolist()})")   # cifar_compress.py:65
        if (f == 4).any():
            raise IndexError(f"symbol outside the table's support or block extent outside [1, 32] x [1, 32] "     # P[i, s] in the reference
                             f"(streams {np.nonzero(f == 4)[0][:8].tolist()})")
        if (f == 2).any():
            raise OverflowError(f"ANS word-stack capacity exhausted (streams {np.nonzero(f == 2)[0][:8].tolist()})")
        if (f != 0).any():
            raise AssertionError(f"ANS stream error flags {np.unique(f).tolist()}")
