"""ORACLE extension (test infrastructure, NOT product code): oracle/blockval.py's block validator with the endorsement policy evaluated
over principal bits and ImplicitMeta nodes.

  SatisfiesPrincipal        bits[i][p] = identity i satisfies principal p, as the caller's MSP answers it (msp/mspimpl.go:483-680);
                            without bits, MSP-member matching of a valid identity, as oracle/blockval.py does (mspimpl.go:501-505)
  cauthdsl NOutOf/SignedBy  common/cauthdsl/cauthdsl.go:24-92 (one `used` array per policy evaluation, policy.go:97-108)
  ImplicitMeta              common/policies/implicitmeta.go:69-103: every sub-policy is evaluated on its own, with its own
                            SignatureSetToValidIdentities and therefore its own `used`; `remaining` counts down from Threshold

Everything before the policy decision -- envelope, header and creator checks, the dispatcher's namespace set, the signature set
(policy.go:365-402) -- is oracle/blockval.validate_tx's: it runs with a policy that every signature set satisfies, and only a
transaction it finds VALID has its signature set rebuilt here and its namespaces' policies evaluated.
"""
import numpy as np

from oracle import blockval as ob
from tools import fabricpb as pb

_ACCEPT = np.array([(0, 0, 0, 0)], np.int32)          # NOutOf(0) over nothing: every signature set satisfies it


def evaluate(nodes, root, signers, satisfies):
    """Policy tree at `root` over the verified, de-duplicated signers; satisfies(signer, p) -> SatisfiesPrincipal(p) == nil."""
    def run(idx, used):
        t, n, first, cnt = [int(x) for x in nodes[idx]]
        if t == 0:                                     # NOutOf (cauthdsl.go:24-58)
            verified = 0
            for c in range(first, first + cnt):
                _used = list(used)
                if run(c, _used):
                    verified += 1
                    used[:] = _used
            return verified >= n
        if t == 2:                                     # ImplicitMeta (implicitmeta.go:69-103)
            remaining = n
            for c in range(first, first + cnt):
                if run(c, [False] * len(signers)):
                    remaining -= 1
                    if remaining == 0:
                        return True
            return remaining == 0
        for i, s in enumerate(signers):                # SignedBy (cauthdsl.go:59-92)
            if used[i] or not satisfies(s, n):
                continue
            used[i] = True
            return True
        return False
    return run(int(root), [False] * len(signers))


class _Roots(dict):
    """The namespace -> root table as validate_tx reads it: every namespace maps to the always-satisfied policy, and the roots it asks
    for are recorded."""

    def __init__(self, real):
        super().__init__({k: 0 for k in real})
        self.real, self.asked = real, []

    def __getitem__(self, k):
        self.asked.append(self.real[k])
        return 0


def _endorsements(env_bytes):
    env = pb.parse(env_bytes, ob.S_ENVELOPE)
    payload = pb.parse(env["payload"], ob.S_PAYLOAD)
    act = pb.parse(pb.parse(payload["data"], ob.S_TX)["actions"][0], ob.S_TXACTION)
    cea = pb.parse(pb.parse(act["payload"], ob.S_CAP)["action"], ob.S_CEA)
    return cea["proposal_response_payload"] or b"", [pb.parse(e, ob.S_ENDORSEMENT) for e in cea["endorsements"]]


def validate_block(block_bytes, identities, channel, nodes, principals, bits=None, policies=None, known=None, verify=ob._verify_fast):
    """oracle/blockval.validate_block with principal bits (bool [n_ids, n_principals], rows in `identities` order) and ImplicitMeta
    nodes (type 2).  bits = None: principals are MSP ids matched as ROLE MEMBER."""
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
        roots = _Roots(policies) if policies is not None else None
        code, txid = ob.validate_tx(d, msp, channel, _ACCEPT, principals, verify, roots)
        if code is None:
            raise NotImplementedError("config transaction at index %d" % t)
        if code == ob.VALID:
            # SignatureSetToValidIdentities (policy.go:365-402), as validate_tx builds it, keeping the identities themselves
            prp, ends = _endorsements(d)
            seen, signers = set(), []
            for e in ends:
                endorser, sig = e["endorser"] or b"", e["signature"] or b""
                idn = msp.deserialize(endorser) if sig else None
                if idn is None or idn[0] in seen or not verify(idn[2], prp + endorser, sig):
                    continue
                seen.add(idn[0])
                signers.append(index[bytes(endorser)])
            for root in (roots.asked if roots is not None else [0]):
                if not evaluate(nodes, root, signers, satisfies):
                    code = ob.ENDORSEMENT_POLICY_FAILURE
                    break
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
