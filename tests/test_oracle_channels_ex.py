"""The batched tickData emulation with identities (orc_channels_tick_data_ex) against the per-channel call it loops over
(orc_channel_tick_data_ex): two sets of oracle channels fed the same subscriptions, updates and ticks must report the same
sends, window starts, self-skip counts and merged ring positions.  CPU only."""
import numpy as np
import pytest

MS = 1_000_000


def test_batched_tick_data_ex_equals_per_channel(oracle):
    rng = np.random.default_rng(31)
    n_ch, n_conn = 300, 40
    batched = oracle.channels(n_ch)
    single = [oracle.channel() for _ in range(n_ch)]
    conn = np.arange(1, n_conn + 1, dtype=np.uint32)
    t = 0
    n_sends = n_update = n_skipped = n_empty = n_multi = 0
    for tick in range(8):
        t += (70 if tick % 3 == 0 else 33) * MS
        # subscribe (or re-subscribe with a new interval) and unsubscribe random pairs
        k = int(rng.integers(100, 400))
        s_ch = rng.integers(0, n_ch, k).astype(np.uint32)
        s_conn = conn[rng.integers(0, n_conn, k)]
        s_iv = rng.choice(np.array([20, 50, 100], np.uint32), k)
        batched.subscribe(s_ch, s_conn, t - 40 * MS, s_iv)
        for c, j, iv in zip(s_ch.tolist(), s_conn.tolist(), s_iv.tolist()):
            single[c].subscribe(j, t - 40 * MS, iv)
        u = int(rng.integers(0, 60))
        u_ch = rng.integers(0, n_ch, u).astype(np.uint32)
        u_conn = conn[rng.integers(0, n_conn, u)]
        batched.unsubscribe(u_ch, u_conn)
        for c, j in zip(u_ch.tolist(), u_conn.tolist()):
            single[c].unsubscribe(j)
        # updates: not time-sorted, half of them from a connection (SkipSelfUpdateFanOut), some cells with none
        m = int(rng.integers(200, 1200))
        m_ch = np.sort(rng.integers(0, n_ch, m)).astype(np.uint32)
        m_arr = (t - rng.integers(0, 120, m) * MS).astype(np.int64)
        m_snd = np.where(rng.random(m) < 0.5, conn[rng.integers(0, n_conn, m)], 7).astype(np.uint32)
        batched.on_update(m_ch, m_arr, m_snd)
        for c, a, snd in zip(m_ch.tolist(), m_arr.tolist(), m_snd.tolist()):
            single[c].on_update(a, snd)
        sends, off, lo, sk, sel_off, sel_pos = batched.tick_data_ex(t, 1 << 16, 1 << 22)
        assert len(sel_off) == len(sends) + 1 and sel_off[0] == 0 and (np.diff(sel_off.astype(np.int64)) >= 0).all()
        assert int(sel_off[-1]) == len(sel_pos) and int(off[-1]) == len(sends)
        for c in range(n_ch):
            want = single[c].tick_data_ex(t)
            b0, b1 = int(off[c]), int(off[c + 1])
            assert b1 - b0 == len(want), c
            for i, d in zip(range(b0, b1), want):
                got = sends[i]
                assert (int(got["conn_id"]), int(got["kind"]), int(got["n_selected"]), int(got["first_sel"]), int(got["last_sel"]),
                        int(got["sel_hash"]), int(got["last_message_index"]), int(got["window_hi"])) == \
                    (d["conn"], d["kind"], d["n"], d["first"], d["last"], d["hash"], d["last_index"], d["window_hi"]), (c, i)
                assert (int(lo[i]), int(sk[i])) == (d["window_lo"], d["self_skipped"]), (c, i)
                assert tuple(sel_pos[int(sel_off[i]):int(sel_off[i + 1])].tolist()) == d["selected"], (c, i)
                n_update += d["kind"] == 1
                n_skipped += d["self_skipped"] > 0
                n_multi += len(d["selected"]) > 1
            n_empty += b1 == b0
        n_sends += len(sends)
    # the comparison covered FULL and UPDATE sends, self-skipped windows, multi-entry selections and channels without sends
    assert n_sends > 1000 and n_update > 300 and n_skipped > 20 and n_multi > 100 and n_empty > 100


def test_batched_tick_data_ex_reports_capacity(oracle):
    """Too small a selection capacity is reported as an error."""
    ch = oracle.channels(4)
    ch.subscribe(np.arange(4), np.full(4, 9), 0, np.full(4, 20))
    sends, *_ = ch.tick_data_ex(30 * MS, 4, 1)  # every pair's first send: FULL, nothing selected
    assert len(sends) == 4 and (sends["kind"] == 0).all()
    ch.on_update(np.array([0, 0, 1]), np.array([35, 36, 37]) * MS, np.full(3, 7))
    with pytest.raises(AssertionError, match="capacity"):
        ch.tick_data_ex(50 * MS, 4, 1)  # cell 0's window [30, 50] ms selects two entries
