"""Minimal protobuf wire-format writer for the Fabric messages on the block-validation path (workload generator side).

Field numbers are those of fabric-protos-go (the reference depends on github.com/trustbloc/fabric-protos-go-ext v0.1.5,
go.mod:14,48; no .proto for these messages exists in the reference tree -- SURVEY.md A.2):

  common.Block{header=1, data=2, metadata=3}      BlockHeader{number=1, previous_hash=2, data_hash=3}
  BlockData{repeated bytes data=1}                Envelope{payload=1, signature=2}
  Payload{header=1, data=2}                       Header{channel_header=1, signature_header=2}
  ChannelHeader{type=1, version=2, timestamp=3, channel_id=4, tx_id=5, epoch=6, extension=7, tls_cert_hash=8}
  SignatureHeader{creator=1, nonce=2}             peer.Transaction{repeated actions=1}
  TransactionAction{header=1, payload=2}          ChaincodeActionPayload{chaincode_proposal_payload=1, action=2}
  ChaincodeEndorsedAction{proposal_response_payload=1, repeated endorsements=2}
  Endorsement{endorser=1, signature=2}            ProposalResponsePayload{proposal_hash=1, extension=2}
  msp.SerializedIdentity{mspid=1, id_bytes=2}
"""


def varint(v: int) -> bytes:
    out = bytearray()
    v &= (1 << 64) - 1
    while True:
        b = v & 0x7F
        v >>= 7
        if v:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def f_bytes(field: int, b: bytes) -> bytes:
    return varint((field << 3) | 2) + varint(len(b)) + bytes(b)


def f_uint(field: int, v: int) -> bytes:
    return varint((field << 3) | 0) + varint(v)


def f_str(field: int, s: str) -> bytes:
    return f_bytes(field, s.encode())


HEADER_TYPE_CONFIG = 1
HEADER_TYPE_CONFIG_UPDATE = 2
HEADER_TYPE_ENDORSER_TRANSACTION = 3


def serialized_identity(mspid: str, id_bytes: bytes) -> bytes:
    return f_str(1, mspid) + f_bytes(2, id_bytes)


def channel_header(htype: int, channel_id: str, tx_id: str, epoch: int = 0, extension: bytes = b"") -> bytes:
    out = f_uint(1, htype) + f_uint(2, 0) + f_str(4, channel_id) + f_str(5, tx_id)
    if epoch:
        out += f_uint(6, epoch)
    if extension:
        out += f_bytes(7, extension)
    return out


def signature_header(creator: bytes, nonce: bytes) -> bytes:
    return (f_bytes(1, creator) if creator else b"") + (f_bytes(2, nonce) if nonce else b"")


def header(chdr: bytes, shdr: bytes) -> bytes:
    return f_bytes(1, chdr) + f_bytes(2, shdr)


def payload(hdr: bytes, data: bytes) -> bytes:
    return f_bytes(1, hdr) + f_bytes(2, data)


def envelope(payload_bytes: bytes, signature: bytes) -> bytes:
    return f_bytes(1, payload_bytes) + (f_bytes(2, signature) if signature else b"")


def endorsement(endorser: bytes, signature: bytes) -> bytes:
    return f_bytes(1, endorser) + f_bytes(2, signature)


def proposal_response_payload(proposal_hash: bytes, extension: bytes) -> bytes:
    return f_bytes(1, proposal_hash) + f_bytes(2, extension)


def chaincode_endorsed_action(prp: bytes, endorsements) -> bytes:
    return f_bytes(1, prp) + b"".join(f_bytes(2, e) for e in endorsements)


def chaincode_action_payload(cc_proposal_payload: bytes, action: bytes) -> bytes:
    return f_bytes(1, cc_proposal_payload) + f_bytes(2, action)


def transaction_action(hdr: bytes, payload_bytes: bytes) -> bytes:
    return f_bytes(1, hdr) + f_bytes(2, payload_bytes)


def transaction(actions) -> bytes:
    return b"".join(f_bytes(1, a) for a in actions)


def block(number: int, envelopes) -> bytes:
    hdr = f_uint(1, number) + f_bytes(2, b"\x00" * 32) + f_bytes(3, b"\x00" * 32)
    data = b"".join(f_bytes(1, e) for e in envelopes)
    return f_bytes(1, hdr) + f_bytes(2, data) + f_bytes(3, b"")


# ---- reader (used by the oracle's block validator) -----------------------------------------------------------

class PbError(Exception):
    pass


def read_varint(b, off):
    """golang/protobuf's decodeVarint: at most 10 bytes, and the 10th may only be 0 or 1 (bit 63); anything else overflows."""
    v = 0
    shift = 0
    while True:
        if off >= len(b):
            raise PbError("truncated varint")
        c = b[off]
        off += 1
        if shift == 63 and c > 1:
            raise PbError("varint overflow")
        v |= (c & 0x7F) << shift
        if not c & 0x80:
            return v, off
        shift += 7


def fields(b):
    """Yields (field_no, wire_type, value) where value is an int (varint / fixed) or a memoryview-like bytes slice."""
    off = 0
    n = len(b)
    while off < n:
        key, off = read_varint(b, off)
        fno, wt = key >> 3, key & 7
        if fno == 0:
            raise PbError("illegal tag 0")
        if wt == 0:
            v, off = read_varint(b, off)
        elif wt == 1:
            if off + 8 > n:
                raise PbError("truncated fixed64")
            v, off = int.from_bytes(b[off:off + 8], "little"), off + 8
        elif wt == 2:
            ln, off = read_varint(b, off)
            if off + ln > n:
                raise PbError("truncated bytes")
            v, off = b[off:off + ln], off + ln
        elif wt == 5:
            if off + 4 > n:
                raise PbError("truncated fixed32")
            v, off = int.from_bytes(b[off:off + 4], "little"), off + 4
        else:
            raise PbError("unsupported wire type %d" % wt)
        yield fno, wt, v


def parse(b, spec):
    """spec: {field_no: (name, kind)} with kind in 'bytes' | 'uint' | 'rep_bytes'.  Unknown fields are skipped; a known
    field with the wrong wire type is an error (as in Go's proto.Unmarshal -- not verified against golang/protobuf v1.3.3, see
    DESIGN.md section 2); later singular occurrences win."""
    out = {name: ([] if kind == "rep_bytes" else None) for name, kind in spec.values()}
    for fno, wt, v in fields(b):
        if fno not in spec:
            continue
        name, kind = spec[fno]
        if kind == "uint":
            if wt != 0:
                raise PbError("wrong wire type for %s" % name)
            out[name] = v
        else:
            if wt != 2:
                raise PbError("wrong wire type for %s" % name)
            if kind == "rep_bytes":
                out[name].append(bytes(v))
            else:
                out[name] = bytes(v)
    return out
