"""The oracle's export of every channel's update buffer (orc_channels_get_rings) against a plain deque restatement of
ChannelData.OnUpdate's buffer half (data.go:149-173) and of how maxFanOutIntervalMs moves (subscription.go:84-86): it grows when a
subscription is created with a longer interval, and never when a kept subscription's interval rises or one is removed.  Floods
past MaxUpdateMsgBufferSize (512) with arrivals out of order, so the eviction rule fires and also declines.  No GPU needed."""
import ctypes as C
from collections import deque

import numpy as np

from tests._oracle import u32p, u64p

MS = 1_000_000
MAX_BUFFER = 512  # MaxUpdateMsgBufferSize, data.go:53-55


class _Channel:
    """data.go:149-173 and subscription.go:43-87, as far as the update buffer depends on them"""

    def __init__(self):
        self.buf = deque()  # (arrival, sender, messageIndex)
        self.msg_index = 0
        self.max_iv = 0
        self.subs = {}

    def subscribe(self, conn, iv):
        if conn in self.subs:  # options merged (subscription.go:43-58): maxFanOutIntervalMs is left alone
            self.subs[conn] = iv
            return
        self.subs[conn] = iv
        self.max_iv = max(self.max_iv, iv)  # subscription.go:84-86

    def unsubscribe(self, conn):
        self.subs.pop(conn, None)

    def on_update(self, arrival, sender):
        self.msg_index += 1
        self.buf.append((arrival, sender, self.msg_index))
        if len(self.buf) > MAX_BUFFER and self.buf[0][0] + self.max_iv * MS < arrival:
            self.buf.popleft()  # one removal per update: the buffer may stay above 512


def _check(got, model):
    n = len(model)
    assert got["off"].tolist() == np.cumsum([0] + [len(m.buf) for m in model]).tolist()
    assert got["msg_index"].tolist() == [m.msg_index for m in model]
    assert got["max_interval_ms"].tolist() == [m.max_iv for m in model]
    want = [e for m in model for e in m.buf]
    assert list(zip(got["arrival"].tolist(), got["sender"].tolist(), got["index"].tolist())) == want
    assert len(got["arrival"]) == int(got["off"][n])


def test_channel_rings_export_matches_the_deque_restatement(oracle):
    rng = np.random.default_rng(31)
    n = 6
    chans = oracle.channels(n)
    model = [_Channel() for _ in range(n)]
    conns = np.arange(100, 140, dtype=np.uint32)
    evictions = kept_rise = declined = 0
    t = 0
    for tick in range(12):
        t += 40 * MS
        # subscriptions: new ones at 20 / 50 / 100 ms, kept ones re-subscribed at a different interval, some removed
        for c in range(n):
            for conn in rng.choice(conns, 6, replace=False):
                conn = int(conn)
                if rng.random() < 0.2 and conn in model[c].subs:
                    chans.unsubscribe([c], [conn])
                    model[c].unsubscribe(conn)
                    continue
                # channel 0 only ever creates 20 ms subscriptions and then raises kept ones to 100 ms
                iv = 20 if c == 0 and conn not in model[c].subs else (100 if c == 0 else int(rng.choice([20, 50, 100])))
                if conn in model[c].subs and iv > model[c].max_iv:
                    kept_rise += 1
                chans.subscribe([c], [conn], t, [iv])
                model[c].subscribe(conn, iv)
        # updates: channels 0-2 get floods (buffer well past 512), the others a few; arrivals not time-sorted
        per = [int(rng.integers(150, 400)) if c < 3 else int(rng.integers(0, 9)) for c in range(n)]
        ch = np.repeat(np.arange(n, dtype=np.uint32), per)
        arr = (t - rng.integers(0, 200, len(ch)) * MS).astype(np.int64)
        snd = np.where(rng.random(len(ch)) < 0.5, rng.choice(conns, len(ch)), 7).astype(np.uint32)
        before = [len(m.buf) for m in model]
        for c, a, s in zip(ch.tolist(), arr.tolist(), snd.tolist()):
            over = len(model[c].buf) + 1 > MAX_BUFFER
            head = model[c].buf[0] if model[c].buf else None
            model[c].on_update(a, s)
            if over and head is not None:
                if model[c].buf[0] is head:
                    declined += 1
                else:
                    evictions += 1
        chans.on_update(ch, arr, snd)
        _check(chans.get_rings(), model)
        assert all(len(m.buf) >= b for m, b in zip(model, before))  # one removal per update at most
    # the eviction rule both fired and declined, a kept pair's interval rose above its channel's maximum, and the maximum stayed
    assert evictions > 100 and declined > 100 and kept_rise > 0
    assert model[0].max_iv == 20 and max(model[0].subs.values()) == 100
    assert len(model[0].buf) > MAX_BUFFER


def test_channel_rings_export_reports_the_total_past_cap(oracle):
    """A buffer smaller than the total: the offsets and the per-channel values are written, the entries are not."""
    chans = oracle.channels(3)
    chans.subscribe([1], [5], 0, [50])
    chans.on_update(np.array([0, 0, 1, 2, 2], np.uint32), np.arange(5, dtype=np.int64) * MS, np.full(5, 9, np.uint32))
    off = np.zeros(4, np.uint64)
    mi = np.zeros(3, np.uint64)
    mx = np.zeros(3, np.uint32)
    arr = np.full(4, -1, np.int64)
    k = chans.L.orc_channels_get_rings(chans._hp(), 3, off.ctypes.data_as(u64p), arr.ctypes.data_as(C.POINTER(C.c_int64)), None, None, 4,
                                       mi.ctypes.data_as(u64p), mx.ctypes.data_as(u32p))
    assert k == 5
    assert off.tolist() == [0, 2, 3, 5] and mi.tolist() == [2, 1, 2] and mx.tolist() == [0, 50, 0]
    assert (arr == -1).all()
