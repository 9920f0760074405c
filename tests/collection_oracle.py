"""ORACLE extension (test infrastructure, NOT product code): tests/policy_oracle.py's block validator with private-data collection
endorsement policies, the table fabgpu_collection_policies installs.

  baseEvaluator.Evaluate        core/common/validation/statebased/validator_keylevel.go:86-142: for the namespace being validated,
                                every public write and public metadata write, then every hashed write and every hashed metadata
                                write of each collection, goes through checkSBAndCCEP(ns, coll, key) (:37-84); with no key-level
                                validation parameter (out of scope here, as on the device) that is CheckCCEPIfNotChecked
  CheckCCEPIfNotChecked         v20.go:105-147: coll != "" -> the collection's policy from CollectionValidationInfo; an empty policy
                                falls through to the chaincode's; coll == "" -> the chaincode's.  nsEPChecked only skips evaluations
                                already made, which cannot change an outcome
  CheckCCEPIfNoEPChecked        v20.go:149-163: the chaincode's policy when no write checked anything
  CollectionValidationInfo      core/chaincode/lifecycle/deployedcc_infoprovider.go:359-394: resolved by the caller into the table
                                {(namespace, collection): root}; a static collection without a policy maps to its chaincode's root.
                                A pair the table does not hold would be read from the ledger: NOT_VALIDATED (254), as the device does

Everything before the policy decision is oracle/blockval.validate_tx's, run through policy_oracle (which reuses it with a policy every
signature set satisfies); the policies are evaluated with policy_oracle.evaluate over the same signer set.
"""
import numpy as np

from oracle import blockval as ob
from tools import fabricpb as pb
import policy_oracle

MAX_COLL = 8            # BD_MAX_COLL: named collections written per transaction the device records


def _results(env_bytes):
    """The TxReadWriteSet bytes of a transaction validate_tx found VALID (so every level on the way parses)."""
    env = pb.parse(env_bytes, ob.S_ENVELOPE)
    payload = pb.parse(env["payload"], ob.S_PAYLOAD)
    chdr = pb.parse(pb.parse(payload["header"], ob.S_HEADER)["channel_header"] or b"", ob.S_CHDR_EXT)
    hext = pb.parse(chdr["extension"] or b"", ob.S_CC_HDR_EXT)
    ccid = (pb.parse(hext["chaincode_id"], ob.S_CCID)["name"] or b"").decode("utf-8", "replace")
    prp, _ = policy_oracle._endorsements(env_bytes)
    cca = pb.parse(pb.parse(prp, ob.S_PRP)["extension"], ob.S_CCACTION)
    return ccid, cca["results"]


def written(results):
    """[(namespace, public: bool, [collection names written])] in read/write-set order.  public: a public write or metadata write
    (validator_keylevel.go:97-111), or a hashed (metadata) write in a collection whose name is empty -- CheckCCEPIfNotChecked(cc, "")
    is the chaincode's policy.  A collection with hashed reads only checks nothing."""
    out = []
    for nsb in pb.parse(results or b"", ob.S_TXRWSET)["ns_rwset"]:
        ns = pb.parse(nsb, ob.S_NSRWSET)
        kv = pb.parse(ns["rwset"] or b"", ob.S_KVRWSET)
        public, colls = len(kv["writes"]) > 0 or len(kv["metadata_writes"]) > 0, []
        for cb in ns["collection_hashed_rwset"]:                                         # :115-137
            c = pb.parse(cb, ob.S_COLLHASHED)
            h = pb.parse(c["hashed_rwset"] or b"", ob.S_HASHEDRWSET)
            if not (h["hashed_writes"] or h["metadata_writes"]):
                continue
            name = (c["collection_name"] or b"").decode("utf-8", "replace")
            if name:
                colls.append(name)
            else:
                public = True
        out.append(((ns["namespace"] or b"").decode("utf-8", "replace"), public, colls))
    return out


def policy_roots(ccid, results, policies, collections):
    """The roots a VALID-so-far transaction must satisfy, or None when one is not in the tables (NOT_VALIDATED).  The dispatcher validates
    the invoked chaincode and every namespace that writes (dispatcher.go:166-221), each with Evaluate above."""
    ns_list = written(results)
    if sum(len(c) for _, _, c in ns_list) > MAX_COLL:
        return None
    by_ns = {n: (p, c) for n, p, c in ns_list}
    order = [ccid] + [n for n, p, c in ns_list if (p or c) and n != ccid]
    roots = []
    for ns in order:
        cc_root = policies[ns] if policies is not None else 0
        public, colls = by_ns.get(ns, (False, []))
        for coll in colls:
            if (ns, coll) not in collections:
                return None
            roots.append(collections[(ns, coll)])
        if public or not colls:                                                          # v20.go:132-146, :149-163
            roots.append(cc_root)
    return roots


def validate_block(block_bytes, identities, channel, nodes, principals, bits=None, policies=None, collections=None, known=None,
                   verify=ob._verify_fast):
    """policy_oracle.validate_block with a collection table {(namespace, collection): root}.  collections = None or empty: no table, which
    is policy_oracle.validate_block itself."""
    if not collections:
        return policy_oracle.validate_block(block_bytes, identities, channel, nodes, principals, bits=bits, policies=policies, known=known,
                                            verify=verify)
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
    flags = np.full(len(data), ob.NOT_VALIDATED, np.uint8)
    txids = [""] * len(data)
    for t, d in enumerate(data):
        roots = policy_oracle._Roots(policies) if policies is not None else None
        code, txid = ob.validate_tx(d, msp, channel, policy_oracle._ACCEPT, principals, verify, roots)
        if code is None:
            raise NotImplementedError("config transaction at index %d" % t)
        if code == ob.VALID:
            ccid, results = _results(d)
            need = policy_roots(ccid, results, policies, collections)
            if need is None:
                code = ob.NOT_VALIDATED
            else:
                # SignatureSetToValidIdentities (policy.go:365-402), as policy_oracle rebuilds it
                prp, ends = policy_oracle._endorsements(d)
                seen, signers = set(), []
                for e in ends:
                    endorser, sig = e["endorser"] or b"", e["signature"] or b""
                    idn = msp.deserialize(endorser) if sig else None
                    if idn is None or idn[0] in seen or not verify(idn[2], prp + endorser, sig):
                        continue
                    seen.add(idn[0])
                    signers.append(index[bytes(endorser)])
                if not all(policy_oracle.evaluate(nodes, r, signers, satisfies) for r in need):
                    code = ob.ENDORSEMENT_POLICY_FAILURE
        flags[t] = code
        if code == ob.VALID:
            txids[t] = txid
    seen = set()
    for t, x in enumerate(txids):                        # markTXIdDuplicates (v20/validator.go:283-297)
        if x:
            if x in seen:
                flags[t] = ob.DUPLICATE_TXID
            else:
                seen.add(x)
    return flags
