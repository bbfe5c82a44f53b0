"""memberlist's probe messages (ping, indirectPingReq, ackResp, nackResp; [U] memberlist/net.go) as gs_wire.h
encodes them for the byte budget of piggybacked broadcasts: known answers, and a cross-check with msgpack-python
packing the same maps in the same field order with go-msgpack's raw strings (use_bin_type=False)."""
import ctypes as C

import msgpack
import pytest

from consul_b200 import _lib

PING, INDIRECT_PING, ACK, NACK = 0, 1, 2, 11


def enc(fn, *args):
    lib = _lib.lib()
    f = getattr(lib, fn)
    n = f(None, 0, *args)
    buf = C.create_string_buffer(n)
    assert f(buf, n, *args) == n
    return buf.raw


def mp(t, fields):
    return bytes([t]) + msgpack.packb(fields, use_bin_type=False)


def test_nack_kat():
    assert enc("gsim_wire_nack", 7) == bytes([NACK, 0x81, 0xA5]) + b"SeqNo" + bytes([7])
    assert enc("gsim_wire_nack", 70000) == bytes([NACK, 0x81, 0xA5]) + b"SeqNo" + bytes([0xCE, 0, 1, 0x11, 0x70])


def test_ack_kat():
    assert enc("gsim_wire_ack", 1, None, 0) == bytes([ACK, 0x82, 0xA5]) + b"SeqNo" + bytes([1, 0xA7]) + b"Payload" + b"\xc0"
    assert enc("gsim_wire_ack", 300, b"\x01ab", 3) == (bytes([ACK, 0x82, 0xA5]) + b"SeqNo" + b"\xcd\x01\x2c" + b"\xa7Payload" +
                                                        b"\xa3\x01ab")


@pytest.mark.parametrize("seq", [0, 127, 128, 65535, 65536, 0xFFFFFFFF])
@pytest.mark.parametrize("src", [True, False])
def test_ping_matches_msgpack(seq, src):
    addr = b"\x0a\x00\x00\x01"
    got = enc("gsim_wire_ping", seq, b"node-1048575", addr if src else None, 4 if src else 0, 8301 if src else 0,
              b"node-17" if src else b"")
    fields = {"SeqNo": seq, "Node": "node-1048575"}
    if src:
        fields.update(SourceAddr=addr, SourcePort=8301, SourceNode="node-17")
    assert got == mp(PING, fields)


@pytest.mark.parametrize("nack", [0, 1])
def test_indirect_ping_matches_msgpack(nack):
    addr = b"\x0a\x00\x00\x02"
    got = enc("gsim_wire_indirect_ping", 65536, addr, 4, 8301, b"node-9", nack, addr, 4, 8301, b"node-12345")
    fields = {"SeqNo": 65536, "Target": addr, "Port": 8301, "Node": "node-9", "Nack": bool(nack),
              "SourceAddr": addr, "SourcePort": 8301, "SourceNode": "node-12345"}
    assert got == mp(INDIRECT_PING, fields)


def test_ack_and_nack_match_msgpack():
    assert enc("gsim_wire_ack", 65536, b"x" * 40, 40) == mp(ACK, {"SeqNo": 65536, "Payload": b"x" * 40})
    assert enc("gsim_wire_ack", 5, None, 0) == mp(ACK, {"SeqNo": 5, "Payload": None})
    assert enc("gsim_wire_nack", 65536) == mp(NACK, {"SeqNo": 65536})


def test_budgets_of_a_1m_pool():
    """What a 1 Mi-member pool's probe messages leave of a 1400-byte UDP buffer (sequence numbers past 2^16, IPv4,
    "node-<id>" names of the pool's capacity): these are the budgets the kernel's piggyback legs use."""
    addr = b"\x0a\x00\x00\x01"
    name = b"node-1048575"
    ping = len(enc("gsim_wire_ping", 65536, name, addr, 4, 8301, name))
    ind = len(enc("gsim_wire_indirect_ping", 65536, addr, 4, 8301, name, 1, addr, 4, 8301, name))
    ack = len(enc("gsim_wire_ack", 65536, None, 0))
    nack = len(enc("gsim_wire_nack", 65536))
    assert (ping, ind, ack, nack) == (85, 111, 22, 13)
    assert 1398 - ack > 1398 - ping > 1398 - ind
