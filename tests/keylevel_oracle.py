"""ORACLE extension (test infrastructure, NOT product code): tests/collection_oracle.py's block validator with key-level validation
parameters (state-based endorsement), the table fabgpu_key_policies installs, and their in-block dependencies.

  checkSBAndCCEP                core/common/validation/statebased/validator_keylevel.go:37-84: for each public write, public metadata
                                write, hashed write and hashed metadata write of the validated namespace (Evaluate, :86-142), the key's
                                validation parameter if it has one -- then SBEPChecked, and not the chaincode or collection policy for
                                that write -- else CheckCCEPIfNotChecked (v20.go:105-147: the collection's policy, or the chaincode's)
  CheckCCEPIfNoEPChecked        v20.go:149-163: the chaincode policy only when no write checked anything -- a namespace without writes
  validation parameter          builtin/v20/validation_logic.go:50-66: a SignaturePolicyEnvelope; one that does not translate is a
                                VSCCExecutionFailureError (the channel halts): the caller maps it to -2, and its writers are 254
  dependencies                  vpmanagerimpl.go:255-289 (ExtractValidationParameterDependency, run by PreValidate for every earlier
                                transaction along extractDependenciesForTx's lenient path, validator_keylevel.go:183-240) registers each
                                (ns, coll, key) a transaction metadata-writes; :196-230 makes a later writer of that key wait for that
                                transaction's VSCC result for the key's namespace, and fail with a policy error (10) if it is nil.

Why "undetermined -> 254" covers exactly the hangs: the result an earlier writer j signals for namespace ns (PostValidate,
validator_keylevel.go:273-276, called by the dispatcher per namespace it validates) exists only if j reached ns's VSCC.  If j's final
flag is VALID, every namespace it validates returned nil.  If it is 10 and j validates one namespace, that namespace -- the written
one -- returned non-nil.  In every other case j either never reached VSCC (rejected before it: the wait never ends), or failed with
several validated namespaces, where the dispatcher returns at the first failure while ranging over a Go map (dispatcher.go:190-217) so
whether ns was reached is not determined by the block -- the reference may wait forever.  Those are 254, and only those.

The lenient path dereferences tx.Actions[0] and cap.Action without checks: a transaction without an action, or whose action payload has
no ChaincodeEndorsedAction, makes the reference's extraction fail hard; no dependency of that block is trusted (254 at the policy stage).
"""
import numpy as np

from oracle import blockval as ob
from tools import fabricpb as pb
import collection_oracle
import policy_oracle

MAX_NEED = 16
S_KVWRITE = {1: ("key", "bytes"), 2: ("is_delete", "uint"), 3: ("value", "bytes")}
S_KVMDWRITE = {1: ("key", "bytes"), 2: ("entries", "rep_bytes")}
S_KVWRITEHASH = {1: ("key_hash", "bytes"), 2: ("is_delete", "uint"), 3: ("value_hash", "bytes"), 4: ("is_purge", "uint")}
S_KVMDWRITEHASH = {1: ("key_hash", "bytes"), 2: ("entries", "rep_bytes")}
S_RESPONSE = {1: ("status", "uint"), 2: ("message", "bytes"), 3: ("payload", "bytes")}


class Untrusted(Exception):
    """the reference's dependency extraction would fail hard on this transaction"""


def writes(results):
    """[(namespace, collection, key, is_metadata)] of a TxReadWriteSet as rwset.FromProtoBytes reads it, or None when it does not parse"""
    out = []
    try:
        for nsb in pb.parse(results or b"", ob.S_TXRWSET)["ns_rwset"]:
            ns = pb.parse(nsb, ob.S_NSRWSET)
            name = bytes(ns["namespace"] or b"")
            kv = pb.parse(ns["rwset"] or b"", ob.S_KVRWSET)
            out += [(name, b"", bytes(pb.parse(w, S_KVWRITE)["key"] or b""), False) for w in kv["writes"]]
            out += [(name, b"", bytes(pb.parse(w, S_KVMDWRITE)["key"] or b""), True) for w in kv["metadata_writes"]]
            for cb in ns["collection_hashed_rwset"]:
                c = pb.parse(cb, ob.S_COLLHASHED)
                coll = bytes(c["collection_name"] or b"")
                h = pb.parse(c["hashed_rwset"] or b"", ob.S_HASHEDRWSET)
                out += [(name, coll, bytes(pb.parse(w, S_KVWRITEHASH)["key_hash"] or b""), False) for w in h["hashed_writes"]]
                out += [(name, coll, bytes(pb.parse(w, S_KVMDWRITEHASH)["key_hash"] or b""), True) for w in h["metadata_writes"]]
    except pb.PbError:
        return None
    return out


def metadata_keys(env_bytes):
    """extractDependenciesForTx (validator_keylevel.go:183-221) + ExtractValidationParameterDependency (vpmanagerimpl.go:255-289): the
    (ns, coll, key) this transaction registers.  Raises Untrusted where the reference dereferences past the end."""
    try:
        env = pb.parse(env_bytes, ob.S_ENVELOPE)
        payload = pb.parse(env["payload"] or b"", ob.S_PAYLOAD)
        if payload["header"] is not None:
            pb.parse(payload["header"], ob.S_HEADER)
        acts = pb.parse(payload["data"] or b"", ob.S_TX)["actions"]
        for a in acts:
            pb.parse(a, ob.S_TXACTION)
        if not acts:
            raise Untrusted()
        cap = pb.parse(pb.parse(acts[0], ob.S_TXACTION)["payload"] or b"", ob.S_CAP)
        if cap["action"] is None:
            raise Untrusted()
        cea = pb.parse(cap["action"], ob.S_CEA)
        for e in cea["endorsements"]:
            pb.parse(e, ob.S_ENDORSEMENT)
        prp = pb.parse(cea["proposal_response_payload"] or b"", ob.S_PRP)
        cca = pb.parse(prp["extension"] or b"", ob.S_CCACTION)
        if cca["response"] is not None:
            pb.parse(cca["response"], S_RESPONSE)
        if cca["chaincode_id"] is not None:
            pb.parse(cca["chaincode_id"], ob.S_CCID)
    except pb.PbError:
        return set()
    ws = writes(cca["results"])
    return {(n, c, k) for n, c, k, md in ws if md} if ws is not None else set()


def policy_roots(ccid, ws, policies, collections, vps):
    """The roots a VALID-so-far transaction must satisfy, or None for NOT_VALIDATED: checkSBAndCCEP per write of each validated namespace
    (the invoked chaincode and every namespace that writes, dispatcher.go:166-221), the chaincode's for a namespace without writes."""
    order = [ccid.encode()]
    for n, _, _, _ in ws:
        if n not in order:
            order.append(n)
    roots = []
    for ns in order:
        cc_root = policies[ns.decode()] if policies is not None else 0
        mine = [w for w in ws if w[0] == ns]
        for _, coll, key, _ in mine:
            cname = (ns.decode(), coll.decode("utf-8", "replace"))
            # a collection the table does not hold may be undefined: the reference then skips the key's parameter
            # (CollConfigNotDefinedError, validator_keylevel.go:53-54) and fails in CheckCCEPIfNotChecked -- not decided here
            if coll and collections and cname not in collections:
                return None
            r = vps.get((ns, coll, key))
            if r == -2:
                return None
            if r is None:
                r = collections[cname] if coll and collections else cc_root
            roots.append(r)
        if not mine:
            roots.append(cc_root)
    roots = list(dict.fromkeys(roots))
    return roots if len(roots) <= MAX_NEED else None


def _key(k):
    ns, coll, key = k
    b = lambda x: x.encode() if isinstance(x, str) else bytes(x)
    return (b(ns), b(coll), b(key))


def validate_block(block_bytes, identities, channel, nodes, principals, bits=None, policies=None, collections=None, vps=None, known=None,
                   verify=ob._verify_fast):
    """collection_oracle.validate_block with key-level validation parameters: vps = {(namespace, collection, key): root in `nodes` or
    -2}; None: no table, which is collection_oracle.validate_block itself."""
    if vps is None:
        return collection_oracle.validate_block(block_bytes, identities, channel, nodes, principals, bits=bits, policies=policies,
                                                 collections=collections, known=known, verify=verify)
    vps = {_key(k): v for k, v in vps.items()}
    msp = ob.Msp(identities, known)
    index = {}
    for k, it in enumerate(identities):
        index.setdefault(bytes(it[0]), k)
    if bits is None:
        satisfies = lambda i, p: bool(identities[i][3]) and identities[i][1] == principals[p]
    else:
        bits = np.asarray(bits, bool)
        satisfies = lambda i, p: bool(bits[i, p])
    blk = pb.parse(block_bytes, ob.S_BLOCK)
    data = pb.parse(blk["data"] or b"", ob.S_BLOCKDATA)["data"]
    untrusted, md = False, []
    for d in data:
        try:
            md.append(metadata_keys(d))
        except Untrusted:
            md.append(set())
            untrusted = True
    flags = np.full(len(data), ob.NOT_VALIDATED, np.uint8)
    n_validated = [0] * len(data)
    # per key, the VSCC results of the metadata writers passed so far (0 = non-nil, 1 = nil, 2 = undetermined): t reads them before its own
    # writes are added, so it sees exactly the writers j < t
    passed = {}
    txids = [""] * len(data)
    for t, d in enumerate(data):
        roots = policy_oracle._Roots(policies) if policies is not None else None
        code, txid = ob.validate_tx(d, msp, channel, policy_oracle._ACCEPT, principals, verify, roots)
        if code is None:
            raise NotImplementedError("config transaction at index %d" % t)
        if code == ob.VALID:
            ccid, results = collection_oracle._results(d)
            ws = writes(results)
            need = None if untrusted or ws is None else policy_roots(ccid, ws, policies, collections, vps)
            if need is None:
                code = ob.NOT_VALIDATED
            else:
                n_validated[t] = len({ccid.encode()} | {w[0] for w in ws})
                prp, ends = policy_oracle._endorsements(d)
                seen, signers = set(), []
                for e in ends:
                    endorser, sig = e["endorser"] or b"", e["signature"] or b""
                    idn = msp.deserialize(endorser) if sig else None
                    if idn is None or idn[0] in seen or not verify(idn[2], prp + endorser, sig):
                        continue
                    seen.add(idn[0])
                    signers.append(index[bytes(endorser)])
                ok = all(policy_oracle.evaluate(nodes, r, signers, satisfies) for r in need)
                code = ob.VALID if ok else ob.ENDORSEMENT_POLICY_FAILURE
                # in-block dependencies: the results of the earlier metadata writers of every key this transaction writes
                res = set().union(*[passed.get((w[0], w[1], w[2]), set()) for w in ws])
                code = ob.NOT_VALIDATED if 2 in res else ob.ENDORSEMENT_POLICY_FAILURE if 1 in res else code
        flags[t] = code
        if code == ob.VALID:
            txids[t] = txid
        st = 1 if code == ob.VALID else 0 if code == ob.ENDORSEMENT_POLICY_FAILURE and n_validated[t] == 1 else 2
        for k in md[t]:
            passed.setdefault(k, set()).add(st)
    seen = set()
    for t, x in enumerate(txids):                        # markTXIdDuplicates (v20/validator.go:283-297), after VSCC
        if x:
            if x in seen:
                flags[t] = ob.DUPLICATE_TXID
            else:
                seen.add(x)
    return flags
