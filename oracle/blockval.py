"""ORACLE (test infrastructure, NOT product code).

CPU restatement of the reference's block validator on the signature path -- what decides a transaction's flag in
TRANSACTIONS_FILTER as far as signatures are concerned:

  TxValidator.Validate / ValidateTx        core/committer/txvalidator/v20/validator.go:182-267,300-455
  validation.ValidateTransaction           core/common/validation/msgvalidation.go:248-320
    validateCommonHeader / ChannelHeader / SignatureHeader   :67-147
    checkSignatureFromCreator              :26-64   (DeserializeIdentity, Validate, Verify)
    protoutil.CheckTxID                    protoutil/proputils.go:357-376
    validateEndorserTransaction            :167-245 (one action; proposal-hash binding, protoutil/txutils.go:431-448)
  KeyLevelValidator.Validate               core/common/validation/statebased/validator_keylevel.go:243-259
                                           (SignedData = prp || endorser per endorsement)
  policies.SignatureSetToValidIdentities   common/policies/policy.go:365-402 (dedup, verify, drop on failure)
  cauthdsl compile (N-out-of / SignedBy)   common/cauthdsl/cauthdsl.go:24-92
  markTXIdDuplicates                       v20/validator.go:283-297

Out of the restated scope, exactly as the reference's own unit tests mock them away (v20/validator_test.go:152-196):
ledger lookups (duplicate tx ids already committed, chaincode definitions), read/write-set checks, key-level policies,
config transactions.  The MSP is a table `serialized identity -> (mspid, public key, Validate() outcome)`, which is what
msp/cache serves in steady state; SatisfiesPrincipal is MSP-member matching (identity.mspid == principal.mspid).

Every signature goes through oracle.bccsp_sw / oracle.fast (the restated bccsp/sw verifier), one at a time in the
reference's order; nothing is shared with the product's batching logic.
"""
import hashlib

import numpy as np

from tools import fabricpb as pb
from . import bccsp_sw as o
from . import fast

# peer.TxValidationCode (fabric-protos-go peer/transaction.pb.go)
VALID, NIL_ENVELOPE, BAD_PAYLOAD, BAD_COMMON_HEADER, BAD_CREATOR_SIGNATURE = 0, 1, 2, 3, 4
INVALID_ENDORSER_TRANSACTION, INVALID_CONFIG_TRANSACTION, UNSUPPORTED_TX_PAYLOAD, BAD_PROPOSAL_TXID, DUPLICATE_TXID = 5, 6, 7, 8, 9
ENDORSEMENT_POLICY_FAILURE, UNKNOWN_TX_TYPE, TARGET_CHAIN_NOT_FOUND = 10, 13, 14
BAD_HEADER_EXTENSION, BAD_CHANNEL_HEADER, BAD_RESPONSE_PAYLOAD, BAD_RWSET, ILLEGAL_WRITESET, INVALID_WRITESET, INVALID_CHAINCODE = 19, 20, 21, 22, 23, 24, 25
NOT_VALIDATED, INVALID_OTHER_REASON = 254, 255

S_BLOCK = {1: ("header", "bytes"), 2: ("data", "bytes"), 3: ("metadata", "bytes")}
S_BLOCKDATA = {1: ("data", "rep_bytes")}
S_ENVELOPE = {1: ("payload", "bytes"), 2: ("signature", "bytes")}
S_PAYLOAD = {1: ("header", "bytes"), 2: ("data", "bytes")}
S_HEADER = {1: ("channel_header", "bytes"), 2: ("signature_header", "bytes")}
S_CHDR = {1: ("type", "uint"), 4: ("channel_id", "bytes"), 5: ("tx_id", "bytes"), 6: ("epoch", "uint")}
S_SHDR = {1: ("creator", "bytes"), 2: ("nonce", "bytes")}
S_TX = {1: ("actions", "rep_bytes")}
S_TXACTION = {1: ("header", "bytes"), 2: ("payload", "bytes")}
S_CAP = {1: ("chaincode_proposal_payload", "bytes"), 2: ("action", "bytes")}
S_CEA = {1: ("proposal_response_payload", "bytes"), 2: ("endorsements", "rep_bytes")}
S_ENDORSEMENT = {1: ("endorser", "bytes"), 2: ("signature", "bytes")}
S_PRP = {1: ("proposal_hash", "bytes"), 2: ("extension", "bytes")}
# the plugin dispatcher's view (core/committer/txvalidator/v20/plugindispatcher/dispatcher.go:102-221)
S_CHDR_EXT = {1: ("type", "uint"), 4: ("channel_id", "bytes"), 5: ("tx_id", "bytes"), 6: ("epoch", "uint"), 7: ("extension", "bytes")}
S_CC_HDR_EXT = {2: ("chaincode_id", "bytes")}                                    # peer.ChaincodeHeaderExtension
S_CCID = {1: ("path", "bytes"), 2: ("name", "bytes"), 3: ("version", "bytes")}   # peer.ChaincodeID
S_CCACTION = {1: ("results", "bytes"), 2: ("events", "bytes"), 3: ("response", "bytes"), 4: ("chaincode_id", "bytes")}   # peer.ChaincodeAction
S_CCEVENT = {1: ("chaincode_id", "bytes"), 2: ("tx_id", "bytes"), 3: ("event_name", "bytes"), 4: ("payload", "bytes")}
S_TXRWSET = {1: ("data_model", "uint"), 2: ("ns_rwset", "rep_bytes")}            # rwset.TxReadWriteSet
S_NSRWSET = {1: ("namespace", "bytes"), 2: ("rwset", "bytes"), 3: ("collection_hashed_rwset", "rep_bytes")}
S_KVRWSET = {1: ("reads", "rep_bytes"), 2: ("range_queries_info", "rep_bytes"), 3: ("writes", "rep_bytes"), 4: ("metadata_writes", "rep_bytes")}
S_COLLHASHED = {1: ("collection_name", "bytes"), 2: ("hashed_rwset", "bytes"), 3: ("pvt_rwset_hash", "bytes")}
S_HASHEDRWSET = {1: ("hashed_reads", "rep_bytes"), 2: ("hashed_writes", "rep_bytes"), 3: ("metadata_writes", "rep_bytes")}


def int32_field(v: int) -> int:
    """A proto3 int32 / enum field as Go decodes it: the varint's low 32 bits, two's complement (ChannelHeader.type = 3 + 2^32
    is 3; -1 sent as a 10-byte varint is -1)."""
    v &= 0xFFFFFFFF
    return v - (1 << 32) if v >= 1 << 31 else v


def identity_id(serialized: bytes, mspid: str):
    """The IdentityIdentifier the reference de-duplicates on (common/policies/policy.go:380-386: Mspid + Id, with
    Id = hex(SHA-256(certificate DER)), msp/identities.go:55-76): two byte-different serializations of ONE certificate (PEM line
    wrapping, trailing whitespace) are the same identity.  Falls back to the serialized bytes when no PEM block parses."""
    import base64
    import re
    try:
        sid = pb.parse(bytes(serialized), {1: ("mspid", "bytes"), 2: ("id_bytes", "bytes")})
        m = re.search(rb"-----BEGIN CERTIFICATE-----(.*?)-----END CERTIFICATE-----", sid["id_bytes"] or b"", re.S)
        if m:
            der = base64.b64decode(b"".join(m.group(1).split()), validate=False)
            return (mspid, hashlib.sha256(der).hexdigest())
    except Exception:
        pass
    return (mspid, bytes(serialized).hex())


class Msp:
    """identities: list of (serialized: bytes, mspid: str, key_xy: 64 bytes, valid: bool).  deserialize -> (dedup id, mspid, xy, valid).
    `known` (optional): the serialized identities the DEVICE's table holds; an identity outside it makes the device hand the
    transaction back (NOT_VALIDATED) -- see validate_tx."""

    def __init__(self, identities, known=None):
        self.by_bytes = {bytes(ser): (identity_id(ser, mspid), mspid, bytes(xy), bool(valid)) for (ser, mspid, xy, valid) in identities}
        self.known = None if known is None else {bytes(k) for k in known}

    def deserialize(self, ser):
        return self.by_bytes.get(bytes(ser))

    def on_device(self, ser):
        return self.known is None or bytes(ser) in self.known


def _verify(xy: bytes, msg: bytes, sig: bytes) -> bool:
    """identity.Verify (msp/identities.go:169-196): SHA-256 then bccsp.Verify; any failure is an error."""
    key = o.P256PublicKey(int.from_bytes(xy[:32], "big"), int.from_bytes(xy[32:], "big"))
    return o.identity_verify(key, msg, sig, "SHA2") is None


def _verify_fast(xy: bytes, msg: bytes, sig: bytes) -> bool:
    st = fast.verify_batch(np.frombuffer(xy, np.uint8).reshape(1, 64), np.zeros(1, np.int32), np.frombuffer(hashlib.sha256(msg).digest(), np.uint8),
                           np.array([0, 32], np.uint32), np.frombuffer(sig, np.uint8) if sig else np.zeros(0, np.uint8), np.array([0, len(sig)], np.uint32))
    return int(st[0]) == o.VALID


def evaluate_policy(nodes, principals, identities_mspid):
    """cauthdsl.compile + evaluator (common/cauthdsl/cauthdsl.go:24-92, policy.go:97-108).
    nodes: int32[k,4] rows (type, n, first_child, n_children); identities_mspid: MSP ids of the valid, deduplicated signers."""
    def run(idx, used):
        t, n, first, cnt = [int(x) for x in nodes[idx]]
        if t == 0:                                   # NOutOf
            verified = 0
            for c in range(first, first + cnt):
                _used = list(used)
                if run(c, _used):
                    verified += 1
                    used[:] = _used
            return verified >= n
        want = principals[n]                          # SignedBy(n)
        for i, mspid in enumerate(identities_mspid):
            if used[i]:
                continue
            if mspid != want:                         # SatisfiesPrincipal: MSP member match
                continue
            used[i] = True
            return True
        return False
    return run(0, [False] * len(identities_mspid))


def evaluate_policy_at(nodes, principals, identities_mspid, root):
    """evaluate_policy with the tree rooted at node `root` (several policies share one node array)."""
    def run(idx, used):
        t, n, first, cnt = [int(x) for x in nodes[idx]]
        if t == 0:
            verified = 0
            for c in range(first, first + cnt):
                _used = list(used)
                if run(c, _used):
                    verified += 1
                    used[:] = _used
            return verified >= n
        want = principals[n]
        for i, mspid in enumerate(identities_mspid):
            if used[i] or mspid != want:
                continue
            used[i] = True
            return True
        return False
    return run(int(root), [False] * len(identities_mspid))


def written_namespaces(results: bytes):
    """rwsetutil.TxRwSet.FromProtoBytes + txWritesToNamespace (dispatcher.go:121-124,166-179,278-300): the namespaces of the
    read/write set in order, each with "writes something"; raises PbError where proto.Unmarshal of a message on that path would.
    (The KVRead / KVWrite entries themselves are not re-parsed: restated scope = what decides the namespace set.)"""
    out = []
    tx = pb.parse(results or b"", S_TXRWSET)
    for nsb in tx["ns_rwset"]:
        ns = pb.parse(nsb, S_NSRWSET)
        kv = pb.parse(ns["rwset"] or b"", S_KVRWSET)
        writes = len(kv["writes"]) > 0 or len(kv["metadata_writes"]) > 0
        for cb in ns["collection_hashed_rwset"]:
            c = pb.parse(cb, S_COLLHASHED)
            h = pb.parse(c["hashed_rwset"] or b"", S_HASHEDRWSET)
            writes = writes or len(h["hashed_writes"]) > 0 or len(h["metadata_writes"]) > 0
        out.append(((ns["namespace"] or b"").decode("utf-8", "replace"), writes))
    return out


def validate_tx(env_bytes, msp: Msp, channel: str, nodes, principals, verify=_verify_fast, policies=None):
    """One transaction -> (code, txid).  Mirrors ValidateTx + ValidateTransaction + the plugin dispatcher + the VSCC signature-policy
    check.  policies: {namespace: root node index} -- the endorsement policy of each chaincode (what GetInfoForValidate returns,
    dispatcher.go:265-277); None = one policy (root 0) for every namespace.  A namespace without an entry, like an identity the
    device table does not hold (Msp.known), cannot be decided by the device: NOT_VALIDATED at the point where it is needed."""
    # zero-length data unmarshals to an empty Envelope (protoutil.GetEnvelopeFromBlock): no header -> BAD_COMMON_HEADER
    try:
        env = pb.parse(env_bytes, S_ENVELOPE)
    except pb.PbError:
        return INVALID_OTHER_REASON, ""               # v20/validator.go:313-320
    # ---- validation.ValidateTransaction ----
    try:
        payload = pb.parse(env["payload"] or b"", S_PAYLOAD)
    except pb.PbError:
        return BAD_PAYLOAD, ""
    try:
        if payload["header"] is None:
            raise pb.PbError("nil header")
        hdr = pb.parse(payload["header"], S_HEADER)
        chdr = pb.parse(hdr["channel_header"] or b"", S_CHDR_EXT)
        shdr = pb.parse(hdr["signature_header"] or b"", S_SHDR)
        chdr["type"] = int32_field(chdr["type"] or 0)
        if chdr["type"] not in (1, 2, 3):
            raise pb.PbError("invalid header type")
        if (chdr["epoch"] or 0) != 0:
            raise pb.PbError("invalid epoch")
        if not shdr["nonce"]:
            raise pb.PbError("invalid nonce")
        if not shdr["creator"]:
            raise pb.PbError("invalid creator")
    except pb.PbError:
        return BAD_COMMON_HEADER, ""
    # checkSignatureFromCreator (msgvalidation.go:26-64)
    if not env["signature"] or not env["payload"]:
        return BAD_CREATOR_SIGNATURE, ""              # "nil arguments"
    if not msp.on_device(shdr["creator"]):
        return NOT_VALIDATED, ""                      # the device cannot deserialize / validate a certificate it was not given
    ident = msp.deserialize(shdr["creator"])
    if ident is None or not ident[3]:
        return BAD_CREATOR_SIGNATURE, ""              # MSP error / certificate not valid
    if not verify(ident[2], env["payload"], env["signature"]):
        return BAD_CREATOR_SIGNATURE, ""
    htype = chdr["type"] or 0
    if htype == 1:
        return None, ""                               # CONFIG: outside the restated scope (configtx validation)
    if htype != 3:
        return UNSUPPORTED_TX_PAYLOAD, ""
    txid = (chdr["tx_id"] or b"").decode("utf-8", "replace")
    if txid != hashlib.sha256(shdr["nonce"] + shdr["creator"]).hexdigest():
        return BAD_PROPOSAL_TXID, ""
    # validateEndorserTransaction (msgvalidation.go:167-245)
    try:
        if payload["data"] is None:
            raise pb.PbError("nil arguments")
        tx = pb.parse(payload["data"], S_TX)
        if len(tx["actions"]) != 1:
            raise pb.PbError("only one action per transaction is supported")
        act = pb.parse(tx["actions"][0], S_TXACTION)
        ashdr = pb.parse(act["header"] or b"", S_SHDR)
        if not ashdr["nonce"] or not ashdr["creator"]:
            raise pb.PbError("invalid signature header")
        cap = pb.parse(act["payload"] or b"", S_CAP)
        if cap["action"] is None:
            raise pb.PbError("nil action")              # the Go code would dereference nil here; treated as invalid
        cea = pb.parse(cap["action"], S_CEA)
        prp = pb.parse(cea["proposal_response_payload"] or b"", S_PRP)
        if hdr["channel_header"] is None or act["header"] is None or cap["chaincode_proposal_payload"] is None:
            raise pb.PbError("nil arguments")
        phash = hashlib.sha256(hdr["channel_header"] + act["header"] + cap["chaincode_proposal_payload"]).digest()
        if phash != (prp["proposal_hash"] or b""):
            raise pb.PbError("proposal hash does not match")
    except pb.PbError:
        return INVALID_ENDORSER_TRANSACTION, ""
    # ---- ValidateTx ----
    if (chdr["channel_id"] or b"").decode("utf-8", "replace") != channel:
        return TARGET_CHAIN_NOT_FOUND, ""
    # ---- plugin dispatcher (plugindispatcher/dispatcher.go:102-221) ----
    try:                                               # nested messages are parsed with their parent (proto.Unmarshal)
        hext = pb.parse(chdr["extension"] or b"", S_CC_HDR_EXT)
        h_ccid = pb.parse(hext["chaincode_id"], S_CCID) if hext["chaincode_id"] is not None else None
    except pb.PbError:
        return BAD_HEADER_EXTENSION, ""
    try:                                               # GetActionFromEnvelope -> GetPayloads (protoutil/txutils.go:20-45)
        if cea["proposal_response_payload"] is None:
            raise pb.PbError("no payload in ChaincodeActionPayload")
        if prp["extension"] is None:
            raise pb.PbError("response payload is missing extension")
        cca = pb.parse(prp["extension"], S_CCACTION)
        r_ccid = pb.parse(cca["chaincode_id"], S_CCID) if cca["chaincode_id"] is not None else None
    except pb.PbError:
        return BAD_RESPONSE_PAYLOAD, ""
    try:
        ns_list = written_namespaces(cca["results"])
    except pb.PbError:
        return BAD_RWSET, ""
    if h_ccid is None or r_ccid is None:
        return INVALID_OTHER_REASON, ""
    ccid = (h_ccid["name"] or b"").decode("utf-8", "replace")
    if ccid == "" or ccid != (r_ccid["name"] or b"").decode("utf-8", "replace") or not (r_ccid["version"] or b""):
        return INVALID_CHAINCODE, ""
    if cca["events"] is not None:
        try:
            ev = pb.parse(cca["events"], S_CCEVENT)
        except pb.PbError:
            return INVALID_OTHER_REASON, ""
        if (ev["chaincode_id"] or b"").decode("utf-8", "replace") != ccid:
            return INVALID_OTHER_REASON, ""
    wr = [ccid]
    seen_ns = set()
    for name, writes in ns_list:
        if name in seen_ns:
            return ILLEGAL_WRITESET, ""
        seen_ns.add(name)
        if writes and name not in wr:
            wr.append(name)
    # ---- VSCC: endorsement policy over the signature set (validator_keylevel.go:243-259, policy.go:365-402) ----
    # One signature set per transaction; the reference rebuilds and re-verifies it for every namespace it validates -- the
    # verdicts cannot differ, so it is evaluated once here and every namespace's policy runs over the same identities.
    try:
        ends = [pb.parse(e, S_ENDORSEMENT) for e in cea["endorsements"]]
    except pb.PbError:
        return INVALID_OTHER_REASON, ""
    roots = []
    for name in wr:
        if policies is None:
            roots.append(0)
        elif name in policies:
            roots.append(policies[name])
        else:
            return NOT_VALIDATED, ""                    # no chaincode definition on the device: the CPU validator looks it up in the ledger
    seen, signer_msps = set(), []
    prp_bytes = cea["proposal_response_payload"] or b""
    for e in ends:
        endorser = e["endorser"] or b""
        if not (e["signature"] or b""):
            continue                                    # can never verify, whoever signed (and needs no identity)
        if not msp.on_device(endorser):
            return NOT_VALIDATED, ""
        idn = msp.deserialize(endorser)
        if idn is None:
            continue                                    # invalid identity: skipped
        if idn[0] in seen:
            continue                                    # de-duplicated (by Mspid + Id) before any signature work
        if not verify(idn[2], prp_bytes + endorser, e["signature"] or b""):
            continue                                    # signature invalid: identity dropped
        seen.add(idn[0])
        if idn[3]:                                      # SatisfiesPrincipal re-validates the identity (msp/mspimpl.go:583-600)
            signer_msps.append(idn[1])
        else:
            signer_msps.append(None)
    for root in roots:
        if not evaluate_policy_at(nodes, principals, signer_msps, root):
            return ENDORSEMENT_POLICY_FAILURE, ""
    return VALID, txid


def validate_block(block_bytes, identities, channel, nodes, principals, verify=_verify_fast, policies=None, known=None):
    """-> uint8 flags (TRANSACTIONS_FILTER), or raises for config transactions (outside the restated scope).
    policies / known: see validate_tx and Msp."""
    msp = Msp(identities, known)
    blk = pb.parse(block_bytes, S_BLOCK)
    data = pb.parse(blk["data"] or b"", S_BLOCKDATA)["data"]
    flags = np.full(len(data), NOT_VALIDATED, np.uint8)
    txids = [""] * len(data)
    for i, d in enumerate(data):
        code, txid = validate_tx(d, msp, channel, nodes, principals, verify, policies)
        if code is None:
            raise NotImplementedError("config transaction at index %d" % i)
        flags[i] = code
        if code == VALID:
            txids[i] = txid
    seen = set()
    for i, t in enumerate(txids):                       # markTXIdDuplicates (v20/validator.go:283-297)
        if not t:
            continue
        if t in seen:
            flags[i] = DUPLICATE_TXID
        else:
            seen.add(t)
    return flags
