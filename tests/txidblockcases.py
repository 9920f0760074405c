"""Test infrastructure (not product code): the envelopes of fabgpu_committed_txids_add_block's cases, each with the id the block store
indexes for it written out (txid_block_oracle restates the rule), and helpers to rebuild a signed envelope with another ChannelHeader or
SignatureHeader."""
import hashlib

from tools import fabricpb as pb

CHANNEL = "txblockchannel"
CREATOR = pb.serialized_identity("Org1MSP", b"-----BEGIN CERTIFICATE-----\ncreator\n-----END CERTIFICATE-----\n")
NONCE = bytes(range(24))
COMPUTED = hashlib.sha256(NONCE + CREATOR).hexdigest()
PLAIN = "ab" * 32


def env(chdr, shdr=None, data=b"\x0a\x00", sig=b"sig"):
    """an envelope of these header bytes (shdr None: the default creator and nonce)"""
    shdr = pb.signature_header(CREATOR, NONCE) if shdr is None else shdr
    return pb.envelope(pb.payload(pb.header(chdr, shdr), data), sig)


def cases():
    """[(name, envelope bytes, the canonical id the block store indexes, or None)]"""
    ch = lambda htype=3, tx_id=PLAIN, epoch=0: pb.channel_header(htype, CHANNEL, tx_id, epoch)
    return [
        ("plain_id", env(ch()), PLAIN),
        ("empty_txid_computed", env(ch(tx_id="")), COMPUTED),
        ("empty_txid_bad_signature_header", env(ch(tx_id=""), shdr=b"\x0a\xff"), None),
        ("empty_txid_signature_header_wrong_wire_type", env(ch(tx_id=""), shdr=pb.f_uint(1, 5)), None),
        ("empty_txid_no_signature_header", pb.envelope(pb.payload(pb.f_bytes(1, ch(tx_id="")), b""), b"s"), hashlib.sha256(b"").hexdigest()),
        ("empty_txid_empty_nonce", env(ch(tx_id=""), shdr=pb.signature_header(CREATOR, b"")), hashlib.sha256(CREATOR).hexdigest()),
        ("empty_txid_empty_creator", env(ch(tx_id=""), shdr=pb.signature_header(b"", NONCE)), hashlib.sha256(NONCE).hexdigest()),
        ("config_type", env(ch(htype=1, tx_id="cd" * 32)), "cd" * 32),
        ("config_type_computed", env(ch(htype=1, tx_id="")), COMPUTED),
        ("header_type_2", env(ch(htype=2, tx_id="ef" * 32)), "ef" * 32),
        ("unknown_header_type", env(ch(htype=77, tx_id="01" * 32)), "01" * 32),
        ("epoch_nonzero", env(ch(tx_id="23" * 32, epoch=5)), "23" * 32),
        ("empty_nonce_with_id", env(ch(tx_id="45" * 32), shdr=pb.signature_header(CREATOR, b"")), "45" * 32),
        ("empty_creator_with_id", env(ch(tx_id="67" * 32), shdr=pb.signature_header(b"", NONCE)), "67" * 32),
        ("bad_signature_header_with_id", env(ch(tx_id="89" * 32), shdr=b"\x0a\xff"), "89" * 32),
        ("uppercase_id", env(ch(tx_id="AB" * 32)), None),
        ("id_63_chars", env(ch(tx_id=PLAIN[:63])), None),
        ("id_65_chars", env(ch(tx_id=PLAIN + "a")), None),
        ("id_non_hex", env(ch(tx_id="g" * 64)), None),
        ("envelope_garbage", b"\x0a\xff\xff", None),
        ("payload_garbage", pb.envelope(b"\x0a\x05ab", b"s"), None),
        ("payload_without_header", pb.envelope(pb.f_bytes(2, b"data"), b"s"), None),
        ("empty_header", pb.envelope(pb.f_bytes(1, b"") + pb.f_bytes(2, b""), b"s"), hashlib.sha256(b"").hexdigest()),
        ("channel_header_garbage", env(b"\x2a\xff"), None),
        ("channel_header_wrong_wire_type", env(pb.f_bytes(1, b"x") + pb.f_str(5, PLAIN)), None),
        ("empty_envelope", b"", None),
        ("repeated_txid_last_wins", env(pb.f_uint(1, 3) + pb.f_str(5, "cd" * 32) + pb.f_str(5, PLAIN)), PLAIN),
    ]


def _rewrite(msg, field, value):
    """msg with every occurrence of length-delimited `field` replaced by one `value` (None: removed), other fields kept as they are"""
    out, done = b"", False
    for f, wt, v in pb.fields(msg):
        if f == field and wt == 2:
            if value is not None and not done:
                out += pb.f_bytes(field, value)
            done = True
            continue
        if wt == 0:
            out += pb.varint(f << 3) + pb.varint(v)
        elif wt == 2:
            out += pb.f_bytes(f, bytes(v))
        else:
            raise ValueError("wire type %d" % wt)
    return out if done or value is None else out + pb.f_bytes(field, value)


def with_txid(envelope, tx_id):
    """the envelope with ChannelHeader.tx_id replaced (the signature is kept, so it no longer verifies)"""
    def last(msg, field):
        return [bytes(v) for f, wt, v in pb.fields(msg) if f == field and wt == 2][-1]
    payload = last(envelope, 1)
    hdr = last(payload, 1)
    chdr = _rewrite(last(hdr, 1), 5, tx_id.encode() if tx_id else None)
    return _rewrite(envelope, 1, _rewrite(payload, 1, _rewrite(hdr, 1, chdr)))
