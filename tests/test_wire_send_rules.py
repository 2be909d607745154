"""The restatement of connection.go's send rules (tests/_wire.py: Send's drop rule, flush's packet split) checked on cases
derived by hand from connection.go, so the GPU framing tests compare against rules that are themselves pinned.  CPU only.

Sizes: MessagePack{channelId = 0x10000, msgType = 8, msgBody = n bytes} is 4 (tag + 3-byte varint) + 2 + 1 + 3 + n = n + 10
bytes for 16384 <= n < 2^21; as a Packet.messages entry it takes 1 + 3 + (n + 10) bytes."""
from tests import _wire as W

CH = 0x10000


def mp(n, ch=CH):
    m = W.MessagePack(channelId=ch, msgType=8, msgBody=b"\x5a" * n)
    assert m.ByteSize() == n + 10  # the hand-derived size above
    return m


def entry(m):
    b = m.SerializeToString()
    n = len(b)
    return bytes([0x0A, (n & 0x7F) | 0x80, ((n >> 7) & 0x7F) | 0x80, n >> 14]) + b


def test_drop_threshold_is_on_the_message_pack():
    # proto.Size(mp) >= MaxPacketSize - PacketHeaderSize = 65530 is dropped (connection.go:73-74)
    packets, dropped = W.flush([mp(65519)])  # 65529: sent, in a packet of 65533 bytes
    assert dropped == 0 and packets == [entry(mp(65519))] and len(packets[0]) == 65533
    packets, dropped = W.flush([mp(65520)])  # 65530: dropped
    assert (packets, dropped) == ([], 1)
    # the entry length of a sent 65529-byte MessagePack is already >= 65530: the rule is not on the entry
    assert len(entry(mp(65516))) == 65530 and W.flush([mp(65516)])[1] == 0


def test_packet_split_at_max_packet_size():
    a = mp(30000)  # entry 30014
    fit, over = mp(35507), mp(35508)  # entries 35521 and 35522: totals 65535 and 65536
    packets, dropped = W.flush([a, fit])
    assert dropped == 0 and packets == [entry(a) + entry(fit)] and len(packets[0]) == 65535
    packets, dropped = W.flush([a, over])
    assert dropped == 0 and packets == [entry(a), entry(over)]
    # the message that overflowed opens the next packet, and later messages join it (flush :648-659, then the next flush)
    small = mp(20000)
    packets, dropped = W.flush([a, over, small])
    assert packets == [entry(a), entry(over) + entry(small)]


def test_dropped_message_in_the_middle():
    a, b = mp(20000), mp(20001)
    packets, dropped = W.flush([a, mp(70000), b])
    assert dropped == 1 and packets == [entry(a) + entry(b)]


def test_connection_with_every_message_dropped_gets_no_packet():
    assert W.flush([mp(65520), mp(70000)]) == ([], 2)
    assert W.flush([]) == ([], 0)


def test_class_entry_is_one_packet_entry_and_omits_zero_fields():
    # channelId 0, empty value: both fields are left out like proto3 Marshal leaves them out
    e = W.class_entry(0, b"", type_url="u", msg_type=8)
    any_ = b"\x0a\x01u"                        # Any{type_url: "u"}
    cdu = b"\x0a" + bytes([len(any_)]) + any_  # ChannelDataUpdateMessage{data}
    m = b"\x20\x08" + b"\x2a" + bytes([len(cdu)]) + cdu
    assert e == b"\x0a" + bytes([len(m)]) + m
    e = W.class_entry(300, b"\x01\x02", type_url="", msg_type=8)
    any_ = b"\x12\x02\x01\x02"
    cdu = b"\x0a" + bytes([len(any_)]) + any_
    m = b"\x08\xac\x02" + b"\x20\x08" + b"\x2a" + bytes([len(cdu)]) + cdu
    assert e == b"\x0a" + bytes([len(m)]) + m


def test_frame_tag():
    assert W.frame(b"\x01" * 300, 1) == b"CH\x01\x2c\x01" + b"\x01" * 300
