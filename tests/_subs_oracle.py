"""Oracle of explicit subscriptions (include/chd_gpu_subs.h): SubscribeToChannel / UnsubscribeFromChannel with ChannelSubscriptionOptions
field presence (subscription.go:34-125), and the interest update's diff over the same pairs (message_spatial.go:82-128), on top of the
CPU oracle's per-channel fan-out state (one oracle channel per cell, orc_channel_subscribe / orc_channel_unsubscribe).

The presence-mask merge is restated here: orc_channel_subscribe merges a re-subscription by replacing the interval and SkipSelf, so
this class hands it the pair's current value for every field the op does not carry.  It also keeps what the fan-out state does not
hold: each pair's dist (CHD_DIST_EXPLICIT until a query produces it) and its options."""
import ctypes as C

import numpy as np

from tests._oracle import OracleChannels

SUB, UNSUB = 0, 1
OPT_INTERVAL, OPT_DELAY, OPT_SKIP_SELF, OPT_SKIP_FIRST = 1, 2, 4, 8
NEW, MERGED, UNSUBSCRIBED, NOT_SUBSCRIBED, ERR_SLOT, ERR_CHANNEL, ERR_CAPACITY = range(7)
DIST_EXPLICIT = 0xFFFFFFFF


class SubsOracle:
    def __init__(self, orc, cells, conn, default_interval_ms=20, default_delay_ms=0, id_start=0x10000, start_ns=None):
        self.orc = orc
        self.cells = cells
        self.ch = OracleChannels(orc, cells)
        self.conn = [int(c) for c in conn]
        self.default_interval_ms, self.default_delay_ms, self.id_start = default_interval_ms, default_delay_ms, id_start
        self.start_ns = np.zeros(cells, np.int64) if start_ns is None else np.asarray(start_ns, np.int64)
        self.pairs = {}  # (slot, cell) -> [dist, interval_ms, skip_self]
        self.cells_of = {}  # slot -> the cells it is subscribed to
        self.pending = set()  # slots with a removal pending

    def _h(self, cell):
        return C.c_void_p(int(self.ch.h[cell]))

    def _sub(self, slot, cell, now_ns, interval, delay, skip_self, skip_first):
        return self.orc.lib.orc_channel_subscribe(self._h(cell), self.conn[slot], int(now_ns - self.start_ns[cell]), int(interval), int(delay),
                                                  int(bool(skip_self)), int(bool(skip_first)))

    def _unsub(self, slot, cell):
        self.orc.lib.orc_channel_unsubscribe(self._h(cell), self.conn[slot])
        del self.pairs[(slot, cell)]
        self.cells_of[slot].discard(cell)

    def _add(self, slot, cell, v):
        self.pairs[(slot, cell)] = v
        self.cells_of.setdefault(slot, set()).add(cell)

    def slot_ok(self, slot):
        return slot < len(self.conn) and self.conn[slot] != 0 and slot not in self.pending

    def apply(self, slot, channel, op, now_ns, present=None, interval=None, delay=None, skip_self=None, skip_first=None, max_pairs=None):
        """One batch in array order -> statuses.  max_pairs: the capacity rule (nothing applied when the result would not fit)."""
        n = len(slot)
        present = np.zeros(n, np.uint8) if present is None else present
        st = np.zeros(n, np.uint8)
        if max_pairs is not None:  # the total after the batch, on a copy of the pair set
            keys = set(self.pairs)
            for i in range(n):
                c = int(channel[i]) - self.id_start
                if not self.slot_ok(int(slot[i])) or not 0 <= c < self.cells:
                    continue
                (keys.discard if op[i] & 1 else keys.add)((int(slot[i]), c))
            if len(keys) > max_pairs:
                for i in range(n):
                    c = int(channel[i]) - self.id_start
                    st[i] = ERR_SLOT if not self.slot_ok(int(slot[i])) else (ERR_CHANNEL if not 0 <= c < self.cells else ERR_CAPACITY)
                return st
        for i in range(n):
            s, c = int(slot[i]), int(channel[i]) - self.id_start
            if not self.slot_ok(s):
                st[i] = ERR_SLOT
                continue
            if not 0 <= c < self.cells:
                st[i] = ERR_CHANNEL
                continue
            p = int(present[i])
            cur = self.pairs.get((s, c))
            if op[i] & 1:  # subscription.go:104-125
                if cur is None:
                    st[i] = NOT_SUBSCRIBED
                else:
                    self._unsub(s, c)
                    st[i] = UNSUBSCRIBED
            elif cur is not None:  # subscription.go:44-57: proto.Merge; delay and SkipFirst only act at creation
                if p & OPT_INTERVAL:
                    cur[1] = int(interval[i])
                if p & OPT_SKIP_SELF:
                    cur[2] = bool(skip_self[i])
                assert self._sub(s, c, now_ns, cur[1], 0, cur[2], False) == 1
                st[i] = MERGED
            else:  # subscription.go:59-87: the SPATIAL defaults, then the fields present
                iv = int(interval[i]) if p & OPT_INTERVAL else self.default_interval_ms
                dl = int(delay[i]) if p & OPT_DELAY else self.default_delay_ms
                ss = bool(skip_self[i]) if p & OPT_SKIP_SELF else True
                sf = bool(skip_first[i]) if p & OPT_SKIP_FIRST else False
                assert self._sub(s, c, now_ns, iv, dl, ss, sf) == 0
                self._add(s, c, [DIST_EXPLICIT, iv, ss])
                st[i] = NEW
        return st

    def interest(self, slot, cells, dists, now_ns, damping):
        """A successful query of `slot` with result cells / dists (message_spatial.go:82-128) -> (new cells, gone cells)."""
        want = dict(zip((int(c) for c in cells), (int(d) for d in dists)))
        have = set(self.cells_of.get(slot, ()))
        gone = sorted(have - set(want))
        for c in gone:
            self._unsub(slot, c)
        new = []
        for c, d in sorted(want.items()):
            iv = damping(d)
            cur = self.pairs.get((slot, c))
            if cur is None:
                assert self._sub(slot, c, now_ns, iv, self.default_delay_ms, True, False) == 0
                self._add(slot, c, [d, iv, True])
                new.append(c)
            else:  # kept: the damping interval and the query's dist; SkipSelf and the fan-out state stay
                cur[0], cur[1] = d, iv
                assert self._sub(slot, c, now_ns, iv, 0, cur[2], False) == 1
        return new, gone

    def remove(self, slot):
        """chd_remove_subscribers as applied by the next interest update: every pair of the slot goes, the slot is free."""
        for c in list(self.cells_of.get(slot, ())):
            self._unsub(slot, c)
        self.conn[slot] = 0
        self.pending.discard(slot)

    def table(self, n_slots):
        """The pairs as chd_get_pairs reports them: off[n_slots + 1], channel, dist, interval (slot, then cell ascending)."""
        keys = sorted(self.pairs)
        off = np.zeros(n_slots + 1, np.uint32)
        np.add.at(off, np.array([s + 1 for s, _ in keys], np.int64), 1) if keys else None
        off = np.cumsum(off).astype(np.uint32)
        ch = np.array([c + self.id_start for _, c in keys], np.uint32)
        dist = np.array([self.pairs[k][0] for k in keys], np.uint32)
        iv = np.array([self.pairs[k][1] for k in keys], np.uint32)
        ss = np.array([self.pairs[k][2] for k in keys], bool)
        return dict(off=off, channel=ch, dist=dist, interval=iv, skip_self=ss, keys=keys)

    def state(self):
        """Fan-out state of every pair in table order -> (last, had_first, last_index)."""
        keys = sorted(self.pairs)
        chan = np.array([c for _, c in keys], np.uint32)
        conn = np.array([self.conn[s] for s, _ in keys], np.uint32)
        last, had, li, found = self.ch.state(chan, conn)
        assert found.all()
        return last, had, li
