"""ORACLE extension (test infrastructure, NOT product code): the v1.4 block validator with the builtin v13 VSCC and chaincode definitions
read from lscc -- what a channel without V2_0Validation runs (core/committer/txvalidator/router.go:43) and what
fabgpu_channel_capability(FABGPU_CAP_V1_3) selects.  Layered over tests/keylevel_oracle.py; file:line refer to the reference tree.

  ValidateTx, ValidateTransaction    v14/validator.go:269-445: unchanged from v2.0 (creator, tx id, proposal hash, TARGET_CHAIN_NOT_FOUND,
                                     config -> 254, UNKNOWN_TX_TYPE), so oracle/blockval.validate_tx runs them.  The one difference
                                     noted: v14 has no plugin dispatcher, and VSCCValidateTx (v14/vscc_validator.go:55-270) takes its place
  chaincode name / version           vscc_validator.go:86-115: empty name, header/action name mismatch, empty version -> 255 (v2.0: 25);
                                     the checks before them (header extension, GetActionFromEnvelope, FromProtoBytes, nil ChaincodeIds)
                                     and the chaincode-event check after them are in the same order as the dispatcher's
  duplicate namespace                :127-132: 23, before any system-chaincode rule
  writes to lscc                     :151-153,176-179: an application chaincode writing lscc -> 23
  writes to vscc / escc / cscc       :155-160,187-190,407-417: an application chaincode writing one -> 23; "writes" is txWritesToNamespace
                                     (:372-403) with V1_3's KeyLevelEndorsement and PrivateChannelData: public writes or metadata writes,
                                     hashed writes or hashed metadata writes
  invoking vscc / escc               :235-238: 23
  invoking lscc                      :230-270 + v13/validation_logic.go:223-231: deploy / upgrade validation, not restated: 254, and the
                                     block is marked (below) -- so is it when the transaction is 254 for any other reason (a creator the
                                     device does not hold, more namespaces than it records): the reference may still accept the upgrade
  invoking qscc / cscc               :240-266,339-366: only the invoked namespace, with its table entry (the caller installs
                                     SignedByAnyMember of the channel's MSP ids); none -> 254; no version check
  application namespaces             :117-149,192-229: the invoked chaincode, then every other written namespace in read/write-set
                                     order; the first failing namespace decides.  Per namespace: GetInfoForValidate -> its table entry
                                     (none: 254, the CPU validator reads lscc); the invoked one's lscc version (:195-208): none -> 254,
                                     another than ChaincodeAction.chaincode_id.version -> EXPIRED_CHAINCODE (17); then its VSCC
  VSCC of namespace ns               builtin/v13 + statebased/v13.go (policyCheckerV13) + validator_keylevel.go:37-142: ns's own writes
                                     only, each against the key's validation parameter if it has one, else the chaincode policy; no
                                     collection policies.  A namespace without writes: its chaincode policy.  With a collection table and
                                     a key table, a written collection the table does not hold is 254, as in v2.0 mode
  signature set                      policy.go:365-402, built when the first namespace's policy is evaluated: an endorser the device does
                                     not hold is then 254 -- after the earlier namespaces' 254 / 17, as on the device
  dependencies                       keylevel_oracle's rule: a writer's result is determined only when it validated one namespace (or is
                                     VALID); a qscc / cscc invocation's never is (it validates only its own namespace, whatever it
                                     metadata-writes), and with a key table such an invocation writing another namespace is 254
  CHAINCODE_VERSION_CONFLICT         v14/validator.go:210-220,487-530: after markTXIdDuplicates, every still-VALID invocation of a chaincode
                                     that a valid upgrade of the block names is 18.  The upgrade is not decided here: in a block where an
                                     lscc invocation is 254, every VALID flag becomes 254.  After the duplicate pass and the
                                     dependency stage, and fed into neither
"""
import numpy as np

from oracle import blockval as ob
from tools import fabricpb as pb
import collection_oracle
import keylevel_oracle
import policy_oracle

EXPIRED_CHAINCODE, CHAINCODE_VERSION_CONFLICT = 17, 18      # fabric-protos-go peer/transaction.proto
MAX_NEED = 16
MAX_NS_SEEN = 8                                             # BD_MAX_NS_SEEN: namespaces of one read/write set the device records


class _LazyEndorsers(ob.Msp):
    """validate_tx's MSP with the endorsers' table check deferred: its first on_device call is the creator's; the later ones are the
    endorsers', answered yes (an unknown one is then skipped) and remembered, since the v1.3 stage asks only when it evaluates a policy."""

    def __init__(self, identities, known):
        super().__init__(identities, known)
        self.calls, self.unknown_endorser = 0, False

    def on_device(self, ser):
        self.calls += 1
        if self.calls == 1:
            return super().on_device(ser)
        self.unknown_endorser = self.unknown_endorser or not super().on_device(ser)
        return True


def _invokes_lscc(env_bytes):
    """The header extension names lscc, on a transaction whose structure parses as far as validateEndorserTransaction's (the levels the
    device's walk reads before the dispatcher's checks; tx id, proposal hash and channel are not needed for that)."""
    try:
        env = pb.parse(env_bytes, ob.S_ENVELOPE)
        payload = pb.parse(env["payload"] or b"", ob.S_PAYLOAD)
        if payload["header"] is None or payload["data"] is None:
            return False
        hdr = pb.parse(payload["header"], ob.S_HEADER)
        chdr = pb.parse(hdr["channel_header"] or b"", ob.S_CHDR_EXT)
        shdr = pb.parse(hdr["signature_header"] or b"", ob.S_SHDR)
        if ob.int32_field(chdr["type"] or 0) != 3 or (chdr["epoch"] or 0) != 0 or not shdr["nonce"] or not shdr["creator"]:
            return False
        acts = pb.parse(payload["data"], ob.S_TX)["actions"]
        if len(acts) != 1:
            return False
        act = pb.parse(acts[0], ob.S_TXACTION)
        ashdr = pb.parse(act["header"] or b"", ob.S_SHDR)
        cap = pb.parse(act["payload"] or b"", ob.S_CAP)
        if not ashdr["nonce"] or not ashdr["creator"] or cap["action"] is None:
            return False
        cea = pb.parse(cap["action"], ob.S_CEA)
        pb.parse(cea["proposal_response_payload"] or b"", ob.S_PRP)
        if hdr["channel_header"] is None or act["header"] is None or cap["chaincode_proposal_payload"] is None:
            return False
        hext = pb.parse(chdr["extension"] or b"", ob.S_CC_HDR_EXT)
        if hext["chaincode_id"] is None:
            return False
        return (pb.parse(hext["chaincode_id"], ob.S_CCID)["name"] or b"") == b"lscc"
    except pb.PbError:
        return False


def _action_version(env_bytes):
    prp, _ = policy_oracle._endorsements(env_bytes)
    cca = pb.parse(pb.parse(prp, ob.S_PRP)["extension"], ob.S_CCACTION)
    return pb.parse(cca["chaincode_id"], ob.S_CCID)["version"] or b""


def validate_block(block_bytes, identities, channel, nodes, principals, bits=None, policies=None, versions=None, collections=None, vps=None,
                   known=None, verify=ob._verify_fast):
    """The v1.4 validator's flags.  policies: {namespace: root} (None: root 0 for every namespace); versions: {namespace: lscc version}
    (None: no versions); collections: the collection table (used only for the undefined-collection rule with a key table); vps: the
    key table as keylevel_oracle takes it (None: none)."""
    vps = None if vps is None else {keylevel_oracle._key(k): v for k, v in vps.items()}
    versions = versions or {}
    if bits is None:
        satisfies = lambda i, p: bool(identities[i][3]) and identities[i][1] == principals[p]
    else:
        bits = np.asarray(bits, bool)
        satisfies = lambda i, p: bool(bits[i, p])
    index = {}
    for k, it in enumerate(identities):
        index.setdefault(bytes(it[0]), k)
    blk = pb.parse(block_bytes, ob.S_BLOCK)
    data = pb.parse(blk["data"] or b"", ob.S_BLOCKDATA)["data"]
    untrusted, md = False, []
    for d in data:
        try:
            md.append(keylevel_oracle.metadata_keys(d) if vps is not None else set())
        except keylevel_oracle.Untrusted:
            md.append(set())
            untrusted = True
    flags = np.full(len(data), ob.NOT_VALIDATED, np.uint8)
    txids = [""] * len(data)
    passed, lscc_seen = {}, False
    for t, d in enumerate(data):
        msp = _LazyEndorsers(identities, known)
        code, txid = ob.validate_tx(d, msp, channel, policy_oracle._ACCEPT, principals, verify, None)
        if code is None:
            raise NotImplementedError("config transaction at index %d" % t)
        if code == ob.INVALID_CHAINCODE:
            code = ob.INVALID_OTHER_REASON
        validated, determined = [], True
        if code == ob.VALID:
            ccid, results = collection_oracle._results(d)
            written = [n for n, w in ob.written_namespaces(results) if w]
            if ccid in ("vscc", "escc"):
                code = ob.ILLEGAL_WRITESET
            elif len(ob.written_namespaces(results)) > MAX_NS_SEEN:
                code = ob.NOT_VALIDATED                  # more namespaces than the device records
            elif ccid == "lscc":
                code = ob.NOT_VALIDATED
            elif ccid in ("qscc", "cscc"):
                validated, determined = [ccid], False
            elif any(n in ("lscc", "vscc", "escc", "cscc") for n in written):
                code = ob.ILLEGAL_WRITESET
            else:
                validated = [ccid] + [n for n in dict.fromkeys(written) if n != ccid]
        if validated:
            code = _vscc(d, ccid, validated, determined, msp, index, nodes, satisfies, policies, versions, collections, vps, untrusted, passed, verify)
        flags[t] = code
        lscc_seen = lscc_seen or (code == ob.NOT_VALIDATED and _invokes_lscc(d))
        if code == ob.VALID:
            txids[t] = txid
        n_val = len(validated)
        st = 1 if code == ob.VALID and determined else 0 if code == ob.ENDORSEMENT_POLICY_FAILURE and n_val == 1 and determined else 2
        for k in md[t]:
            passed.setdefault(k, set()).add(st)
    seen = set()
    for t, x in enumerate(txids):                        # markTXIdDuplicates (v14/validator.go:210-215)
        if x and flags[t] == ob.VALID:
            if x in seen:
                flags[t] = ob.DUPLICATE_TXID
            else:
                seen.add(x)
    if lscc_seen:                                        # v14/validator.go:216-220,487-530, not decided here
        flags[flags == ob.VALID] = ob.NOT_VALIDATED
    return flags


def _vscc(d, ccid, validated, app, msp, index, nodes, satisfies, policies, versions, collections, vps, untrusted, passed, verify):
    """The namespaces in order (rows 6-9 above); then the in-block dependency rule on the result."""
    ws = []
    if vps is not None:
        ws = keylevel_oracle.writes(collection_oracle._results(d)[1])
        if untrusted or ws is None:
            return ob.NOT_VALIDATED
        if not app and any(w[0] != ccid.encode() for w in ws):
            return ob.NOT_VALIDATED
    signers = None
    code = ob.VALID
    for i, ns in enumerate(validated):
        if policies is not None and ns not in policies:
            return ob.NOT_VALIDATED
        cc_root = policies[ns] if policies is not None else 0
        if i == 0 and app:
            v = versions.get(ns, "") if policies is not None else ""
            if not v:
                return ob.NOT_VALIDATED
            if v.encode() != bytes(_action_version(d)):
                return EXPIRED_CHAINCODE
        roots = []
        mine = [w for w in ws if w[0] == ns.encode()]
        for _, coll, key, _ in mine:
            if coll and collections and (ns, coll.decode("utf-8", "replace")) not in collections:
                return ob.NOT_VALIDATED
            r = vps.get((ns.encode(), coll, key))
            if r == -2:
                return ob.NOT_VALIDATED
            roots.append(cc_root if r is None else r)
        if not mine:
            roots.append(cc_root)
        roots = list(dict.fromkeys(roots))
        if len(roots) > MAX_NEED:
            return ob.NOT_VALIDATED
        if signers is None:
            if msp.unknown_endorser:
                return ob.NOT_VALIDATED
            prp, ends = policy_oracle._endorsements(d)
            seen, signers = set(), []
            for e in ends:
                endorser, sig = e["endorser"] or b"", e["signature"] or b""
                idn = msp.deserialize(endorser) if sig else None
                if idn is None or idn[0] in seen or not verify(idn[2], prp + endorser, sig):
                    continue
                seen.add(idn[0])
                signers.append(index[bytes(endorser)])
        if not all(policy_oracle.evaluate(nodes, r, signers, satisfies) for r in roots):
            code = ob.ENDORSEMENT_POLICY_FAILURE
            break
    if vps is not None:                                  # keylevel_oracle's dependency rule over the transaction's writes
        res = set().union(*[passed.get((w[0], w[1], w[2]), set()) for w in ws])
        code = ob.NOT_VALIDATED if 2 in res else ob.ENDORSEMENT_POLICY_FAILURE if 1 in res else code
    return code
