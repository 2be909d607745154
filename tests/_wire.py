"""Wire messages of the fan-out path, built at run time with the protobuf runtime (no protoc in the image):
channeldpb.Packet / MessagePack / ChannelDataUpdateMessage (pkg/channeldpb/channeld.proto:10-34,333-340) and a channel data
message shaped like internal/testpb/test.proto's TestChannelDataMessage (text, num) extended with a repeated and a map field so
that every merge rule (last scalar wins, lists append, map entries override) is exercised.  Test infrastructure."""
from google.protobuf import any_pb2, descriptor_pb2, descriptor_pool, message_factory

_F = descriptor_pb2.FieldDescriptorProto


def _field(m, name, num, typ, label=_F.LABEL_OPTIONAL, type_name=None):
    f = m.field.add()
    f.name, f.number, f.type, f.label = name, num, typ, label
    if type_name:
        f.type_name = type_name
    return f


def _build():
    pool = descriptor_pool.Default()
    fd = descriptor_pb2.FileDescriptorProto()
    fd.name, fd.package, fd.syntax = "chd_test_wire.proto", "chdtest", "proto3"
    fd.dependency.append("google/protobuf/any.proto")
    mp = fd.message_type.add()
    mp.name = "MessagePack"
    _field(mp, "channelId", 1, _F.TYPE_UINT32)
    _field(mp, "broadcast", 2, _F.TYPE_UINT32)
    _field(mp, "stubId", 3, _F.TYPE_UINT32)
    _field(mp, "msgType", 4, _F.TYPE_UINT32)
    _field(mp, "msgBody", 5, _F.TYPE_BYTES)
    pk = fd.message_type.add()
    pk.name = "Packet"
    _field(pk, "messages", 1, _F.TYPE_MESSAGE, _F.LABEL_REPEATED, ".chdtest.MessagePack")
    cdu = fd.message_type.add()
    cdu.name = "ChannelDataUpdateMessage"
    _field(cdu, "data", 1, _F.TYPE_MESSAGE, type_name=".google.protobuf.Any")
    _field(cdu, "contextConnId", 2, _F.TYPE_UINT32)
    d = fd.message_type.add()
    d.name = "TestChannelDataMessage"
    _field(d, "text", 1, _F.TYPE_STRING)
    _field(d, "num", 2, _F.TYPE_UINT32)
    _field(d, "list", 3, _F.TYPE_STRING, _F.LABEL_REPEATED)
    kv = d.nested_type.add()
    kv.name = "KvEntry"
    kv.options.map_entry = True
    _field(kv, "key", 1, _F.TYPE_UINT32)
    _field(kv, "value", 2, _F.TYPE_STRING)
    _field(d, "kv", 4, _F.TYPE_MESSAGE, _F.LABEL_REPEATED, ".chdtest.TestChannelDataMessage.KvEntry")
    any_pb2.Any()  # make sure any.proto is in the default pool
    pool.Add(fd)
    get = lambda n: message_factory.GetMessageClass(pool.FindMessageTypeByName("chdtest." + n))  # noqa: E731
    return get("Packet"), get("MessagePack"), get("ChannelDataUpdateMessage"), get("TestChannelDataMessage")


Packet, MessagePack, ChannelDataUpdateMessage, TestChannelDataMessage = _build()
TYPE_URL = "type.googleapis.com/chdtest.TestChannelDataMessage"
MSG_CHANNEL_DATA_UPDATE = 8  # channeld.proto:121

# ---- connection.go's send rules, restated with the protobuf runtime measuring every size
MAX_PACKET_SIZE = 0x00FFFF  # connection.go:27
PACKET_HEADER_SIZE = 5      # connection.go:28


def message_pack(channel_id, value, type_url=TYPE_URL, msg_type=MSG_CHANNEL_DATA_UPDATE):
    """The MessagePack Send builds for a CHANNEL_DATA_UPDATE whose Any.value is `value` (data.go:293-318, connection.go:58-71)."""
    body = ChannelDataUpdateMessage(data=any_pb2.Any(type_url=type_url, value=value)).SerializeToString()
    return MessagePack(channelId=channel_id, msgType=msg_type, msgBody=body)


def class_entry(channel_id, value, type_url=TYPE_URL, msg_type=MSG_CHANNEL_DATA_UPDATE):
    """The bytes of that MessagePack as one Packet.messages entry: a Packet holding only it, serialized."""
    return Packet(messages=[message_pack(channel_id, value, type_url, msg_type)]).SerializeToString()


def flush(mps):
    """One connection's MessagePacks in queue order -> (serialized packets, number dropped).
    Send (connection.go:73-77) drops a MessagePack of proto.Size >= MaxPacketSize - PacketHeaderSize; flush (:640-660) appends
    to the packet and, when proto.Size(packet) then exceeds MaxPacketSize, takes the message back out and opens the next
    packet with it."""
    packets, cur, dropped = [], Packet(), 0
    for mp in mps:
        if mp.ByteSize() >= MAX_PACKET_SIZE - PACKET_HEADER_SIZE:
            dropped += 1
            continue
        cur.messages.append(mp)
        if cur.ByteSize() > MAX_PACKET_SIZE:
            del cur.messages[-1]
            packets.append(cur.SerializeToString())
            cur = Packet(messages=[mp])
    if len(cur.messages):
        packets.append(cur.SerializeToString())
    return packets, dropped


def frame(packet, compression_type=0):
    """'C' 'H' size_hi size_lo compressionType + body (connection.go:684-688)."""
    assert len(packet) <= MAX_PACKET_SIZE
    return bytes([67, 72, len(packet) >> 8, len(packet) & 0xFF, compression_type]) + packet
