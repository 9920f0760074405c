"""ORACLE extension (test infrastructure, NOT product code): the ids the block store indexes for a committed block, and the ledger check of a
sequence of blocks in which each block sees the ids of every block before it (fabgpu_committed_txids_add_block).

  GetOrComputeTxIDFromEnvelope   protoutil/txutils.go:485-515
      UnmarshalEnvelope -> UnmarshalPayload -> a nil Payload.Header fails -> UnmarshalChannelHeader(Header.ChannelHeader);
      ChannelHeader.TxId != "" is the id (type, epoch and channel are not looked at, the signature header is not read);
      else UnmarshalSignatureHeader(Header.SignatureHeader) and ComputeTxID(nonce, creator) = hex(SHA-256(nonce || creator))
      (protoutil/proputils.go), with an empty nonce or creator as well.  Every error gives "".
  addDataBytesAndConstructTxIndexInfo   common/ledger/blkstorage/block_serialization.go:95-115
      calls it for every envelope of the block, logs an error and keeps the "" id.
  indexBlock (Index3)                   common/ledger/blkstorage/blockindex.go:112-138
      puts one txid-index entry per transaction, whatever its validation flag, under constructTxIDKey(txID, blkNum, txNum).
      GetTransactionByID then finds the id, so a later transaction carrying it is a ledger duplicate (txid_oracle).

The messages are parsed with tools/fabricpb under the schemas the block oracle uses for the same messages (the walk's selections), so
this module and the validator read one envelope alike.  The committed tx-id set keeps canonical ids only (64 characters of [0-9a-f]);
a computed id always is one, and an "" id or any other form can never equal the id of a transaction that reaches the ledger check.
"""
import hashlib

from oracle import blockval as ob
from tools import fabricpb as pb
import txid_oracle

_HEX = set(b"0123456789abcdef")


def block_store_id(env_bytes):
    """GetOrComputeTxIDFromEnvelope: the id as bytes, b"" where any unmarshal fails"""
    try:
        env = pb.parse(env_bytes, ob.S_ENVELOPE)
        payload = pb.parse(env["payload"] or b"", ob.S_PAYLOAD)
        if payload["header"] is None:                                    # Payload.Header == nil
            return b""
        hdr = pb.parse(payload["header"], ob.S_HEADER)
        chdr = pb.parse(hdr["channel_header"] or b"", ob.S_CHDR_EXT)
        if chdr["tx_id"]:
            return bytes(chdr["tx_id"])
        shdr = pb.parse(hdr["signature_header"] or b"", ob.S_SHDR)
    except pb.PbError:
        return b""
    return hashlib.sha256(bytes(shdr["nonce"] or b"") + bytes(shdr["creator"] or b"")).hexdigest().encode()


def canonical(id_bytes):
    return len(id_bytes) == 64 and set(id_bytes) <= _HEX


def indexed_ids(envelopes):
    """The canonical ids the block store indexes for a block of these envelopes, as str, in order of first occurrence"""
    out = {}
    for e in envelopes:
        i = block_store_id(e)
        if canonical(i):
            out.setdefault(i.decode(), None)
    return list(out)


def sequence(oracle_fn, blocks, installed=None):
    """[oracle_fn(block) with the ledger check] for each block of `blocks`, each seeing the committed table `installed` ({id str: kind})
    plus, with kind 0, the ids of every block before it.  blocks: [(block argument, envelopes)].  A kind-1 id given again by a block keeps
    kind 1 (the larger kind wins)."""
    table = dict(installed or {})
    out = []
    for arg, envs in blocks:
        out.append(txid_oracle.committed(oracle_fn, arg, committed=dict(table)))
        for i in indexed_ids(envs):
            table[i] = max(table.get(i, 0), 0)
    return out


def after(installed, blocks_envs):
    """the table {id str: kind} after installing `installed` and adding the ids of each block of envelopes in turn"""
    table = dict(installed or {})
    for envs in blocks_envs:
        for i in indexed_ids(envs):
            table[i] = max(table.get(i, 0), 0)
    return table
