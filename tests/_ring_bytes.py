"""A plain restatement of byte-carrying device rings (include/chd_gpu_ring_bytes.h) for the tests: one cell's buffer as a deque
with an entry slab of `cap` entries and a byte slab of `bcap` bytes, ChannelData.OnUpdate's 512 / maxFanOutIntervalMs rule
(data.go:149-173), and where the slab cursors go, so that a test can assert which paths a case took.  Also the bytes the tests
give each update: a function of (cell, msgIndex), so the expected bytes of any live entry follow from chd_get_rings."""
from collections import deque

import numpy as np

MS = 1_000_000
MAX_BUFFER = 512  # MaxUpdateMsgBufferSize (data.go:53-55)


class ByteRing:
    def __init__(self, cap, bcap):
        self.cap, self.bcap = cap, bcap
        self.b = self.e = 0    # live entries [b, e) of the entry slab
        self.bb = self.be = 0  # live bytes [bb, be) of the byte slab
        self.ents = deque()    # (arrival, sender, msgIndex, bytes), oldest first
        self.mi = 0
        self.drops = self.slides = self.evictions = 0
        self.byte_slides = []  # the shift of every byte slide

    def _pop(self):
        self.bb += len(self.ents.popleft()[3])
        self.b += 1

    def append(self, t, sender, data, max_interval_ms):
        """one update -> the entries it dropped (CHD_OVF_RING)"""
        L = len(data)
        assert L <= self.bcap
        dropped = 0
        if self.e == self.cap:  # the entry slab's tail is at its end: slide, dropping the oldest entry of a full slab
            if self.e - self.b == self.cap:
                self._pop()
                dropped += 1
            self.slides += 1
            self.b, self.e = 0, self.e - self.b
        while self.be - self.bb + L > self.bcap:  # the byte slab cannot take L more bytes
            self._pop()
            dropped += 1
        if self.be + L > self.bcap:  # no room at the byte tail: slide the live bytes to the slab start
            self.byte_slides.append(self.bb)
            self.be -= self.bb
            self.bb = 0
        self.mi += 1
        self.ents.append((int(t), int(sender), self.mi, bytes(data)))
        self.e += 1
        self.be += L
        if self.e - self.b > MAX_BUFFER and self.ents[0][0] + int(max_interval_ms) * MS < t:
            self._pop()
            self.evictions += 1
        self.drops += dropped
        return dropped

    def live_bytes(self):
        return self.be - self.bb


def entry_bytes(cell, index, max_len=23):
    """the serialized updateMsg the tests give update `index` (msgIndex) of `cell`: 0 .. max_len bytes, a function of both"""
    h = (int(cell) * 0x9E3779B1 + int(index) * 0x85EBCA77) & 0xFFFFFFFF
    n = h % (max_len + 1)
    return bytes(((h >> 8) + 31 * i + int(index)) & 0xFF for i in range(n))


def update_bytes(cells, indices, max_len=23):
    """the bytes of updates (cell, msgIndex) -> (byte_off u64 [n + 1], data u8)"""
    parts = [entry_bytes(c, i, max_len) for c, i in zip(np.asarray(cells).tolist(), np.asarray(indices).tolist())]
    off = np.zeros(len(parts) + 1, np.uint64)
    off[1:] = np.cumsum([len(p) for p in parts], dtype=np.uint64)
    return off, np.frombuffer(b"".join(parts), np.uint8).copy()


def msg_indices(upd_off, msg_index_before):
    """the msgIndex each update of a CSR by cell gets: the cell's msgIndex before the append, plus its rank within the cell"""
    upd_off = np.asarray(upd_off, np.int64)
    n_cell = np.diff(upd_off)
    cell = np.repeat(np.arange(len(n_cell)), n_cell)
    rank = np.arange(int(upd_off[-1])) - upd_off[:-1][cell]
    return cell, np.asarray(msg_index_before, np.int64)[cell] + 1 + rank
