"""Test infrastructure (not product code): a channel whose MSPs use NodeOUs, the principal bits its identities carry, and policy trees
in the device's node layout.

A caller of fabgpu_msp_principal_bits fills bit (i, p) from its own MSP, identity.SatisfiesPrincipal(principal p) == nil.  Here that answer
is computed by the rules of the reference's MSP at version 1.4.2 with NodeOUs enabled (msp/mspimpl.go):
  ROLE MEMBER                     Validate()                                                     :501-505
  ROLE PEER / CLIENT              Validate() and the identity carries that node OU                :514-525, hasOURole :335-379
  ROLE ORDERER                    Validate() and the orderer OU                                   :657-666
  ROLE ADMIN                      listed among the MSP's admin certificates (no Validate()), or   :638-656, isInAdmins :674-680
                                  Validate() and the admin OU
  IDENTITY                        DeserializeIdentity(principal) under the identity's MSP (same MSP id) and the same certificate;
                                  then the principal's Validate()                                 :529-541
Every ROLE principal first requires the principal's MSP id to be the identity's (:494-496, :617-619).
"""
import functools

import numpy as np

from oracle import blockval as ob
from tools import blockgen

ROLES = ("member", "peer", "client", "admin", "orderer")


def cert_id(ident):
    """The certificate an identity carries (hex SHA-256 of its DER): two serializations of one certificate share it."""
    return ob.identity_id(ident.serialized, ident.mspid)[1]


class NodeOUNetwork(blockgen.Network):
    """blockgen.Network whose identities carry node OUs.  Per org: peers_per_org peers (the first is blockgen's peer, also present in
    its second serialization), clients_per_org clients, one identity with the admin OU, one listed among the MSP's admin certificates
    whose Validate() fails (an expired admin certificate: mspimpl.go:674-680 does not re-validate listed admins), and one orderer.
    blockgen's invalid certificate is a peer whose Validate() fails.  Transactions are created by the clients."""

    def __init__(self, n_orgs=4, peers_per_org=2, clients_per_org=2, seed=0x0DE0, channel="fabgpu-channel"):
        per_org = (peers_per_org - 1) + clients_per_org + 3
        super().__init__(n_orgs=n_orgs, n_clients=n_orgs * per_org, seed=seed, channel=channel)
        pool = self.clients                                   # pool[k * n_orgs + o] belongs to org o

        def take(k):
            return [pool[k * n_orgs + o] for o in range(n_orgs)]
        self.org_peers = [[p] for p in self.peers]
        extra = []
        for k in range(peers_per_org - 1):
            for o, p in enumerate(take(k)):
                self.org_peers[o].append(p); extra.append(p)
        k0 = peers_per_org - 1
        clients = [c for k in range(clients_per_org) for c in take(k0 + k)]
        self.admins = take(k0 + clients_per_org)
        self.admins_listed = [blockgen.Identity(i.mspid, i.priv_index, i.xy, i.cert_pem, valid=False) for i in take(k0 + clients_per_org + 1)]
        self.orderers = take(k0 + clients_per_org + 2)
        self.clients = clients
        self.ou = {}
        for i in self.peers + self.peers_alt + extra + [self.invalid_cert]:
            self.ou[i.serialized] = "peer"
        for i, role in [(c, "client") for c in clients] + [(a, "admin") for a in self.admins] + [(a, "client") for a in self.admins_listed] + \
                [(o, "orderer") for o in self.orderers]:
            self.ou[i.serialized] = role
        self.admin_certs = {(i.mspid, cert_id(i)) for i in self.admins_listed}
        self.msp_table = self.peers + self.clients + [self.invalid_cert] + self.peers_alt + extra + self.admins + self.admins_listed + self.orderers

    def identities(self):
        return [(i.serialized, i.mspid, i.xy, i.valid) for i in self.msp_table]


def role(mspid, r):
    """A ROLE principal, e.g. role("Org1MSP", "peer") for 'Org1MSP.peer'."""
    assert r in ROLES
    return ("role", mspid, r)


def identity_principal(ident):
    return ("identity", ident.mspid, cert_id(ident))


def principal_name(p):
    """The string the device is given for principal p (it is only matched as an MSP id when no bits are installed)."""
    return "%s.%s" % (p[1], p[2]) if p[0] == "role" else "%s.identity.%s" % (p[1], p[2][:16])


def satisfies(net, ident, p):
    """identity.SatisfiesPrincipal(p) == nil by the rules in the module docstring."""
    if p[1] != ident.mspid:
        return False
    if p[0] == "identity":
        return cert_id(ident) == p[2] and ident.valid
    r = p[2]
    if r == "member":
        return ident.valid
    if r == "admin" and (ident.mspid, cert_id(ident)) in net.admin_certs:
        return True
    return ident.valid and net.ou.get(ident.serialized) == r


def principal_bits(net, principals):
    """bool [len(net.msp_table), len(principals)]: what a caller hands fabgpu_msp_principal_bits."""
    return np.array([[satisfies(net, i, p) for p in principals] for i in net.msp_table], bool).reshape(len(net.msp_table), len(principals))


def member_roles_for(net, principals):
    """For blockgen.Network (no node OUs of its own): peers and their second serializations are peers, everyone else a client."""
    net.ou = {i.serialized: "client" for i in net.msp_table}
    for i in net.peers + net.peers_alt + [net.invalid_cert]:
        net.ou[i.serialized] = "peer"
    net.admin_certs = set()
    return principal_bits(net, principals)


# ---- policy trees ----------------------------------------------------------------------------------------------------------------
# A tree is ("signed_by", p) | ("n_of", n, [trees]) | ("meta", threshold, [trees]); forest() lays trees out as (type, n, first_child,
# n_children) rows, children contiguous.

def signed_by(p):
    return ("signed_by", p)


def n_of(n, kids):
    return ("n_of", n, list(kids))


def implicit_meta(rule, subs):
    """ImplicitMeta over sub-policies with NewImplicitMetaPolicy's threshold (implicitmeta.go:44-58)."""
    subs = list(subs)
    t = {"ANY": 1, "ALL": len(subs), "MAJORITY": len(subs) // 2 + 1}[rule]
    return ("meta", 0 if not subs else t, subs)


REJECT = ("n_of", 1, [])        # the policy GetPolicy returns for a sub-policy an org lacks: NOutOf(1) over nothing


def forest(trees):
    """-> (nodes int32 [k, 4], root index of each tree)."""
    rows, roots = [], []

    def fill(t, at):
        if t[0] == "signed_by":
            rows[at] = (1, t[1], 0, 0)
            return
        first = len(rows)
        rows.extend([None] * len(t[2]))
        rows[at] = (0 if t[0] == "n_of" else 2, t[1], first, len(t[2]))
        for k, kid in enumerate(t[2]):
            fill(kid, first + k)
    for t in trees:
        roots.append(len(rows)); rows.append(None)
        fill(t, roots[-1])
    return np.array(rows, np.int32).reshape(-1, 4), roots


def stock_endorsement(n_orgs, rule="MAJORITY"):
    """/Channel/Application/Endorsement of a stock channel: ImplicitMeta '<rule> Endorsement' over each org's Endorsement policy
    OR('OrgN.peer') (configtx.yaml).  -> (principals, tree)."""
    principals = [role("Org%dMSP" % (o + 1), "peer") for o in range(n_orgs)]
    return principals, implicit_meta(rule, [n_of(1, [signed_by(o)]) for o in range(n_orgs)])


# ---- the cases both the host build and the device are held to ----------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def network(n_orgs=4):
    return NodeOUNetwork(n_orgs=n_orgs)


def policy_cases():
    """[(name, n_orgs, trees, principals, use_bits, policies, txs)].  trees: policy trees laid out by forest(); policies: {namespace: tree
    index} or None (tree 0 for every namespace); principals: descriptors (role(), identity_principal()) or, without bits, MSP ids;
    txs: [(endorsers, written namespaces or None, expected code)].  Every expected code is written out, not computed."""
    V, F = ob.VALID, ob.ENDORSEMENT_POLICY_FAILURE
    out = []
    for n in (2, 3, 4):
        net = network(n)
        P, maj = net.org_peers, n // 2 + 1
        minority = [P[o][0] for o in range(maj - 1)]
        principals, tree = stock_endorsement(n)
        txs = [([P[o][0] for o in range(maj)], V), ([P[o][1] for o in range(maj)], V), ([P[o][0] for o in range(n)], V),
               (minority, F), (minority + [P[0][0]], F), (minority + [net.peers_alt[0]], F), (minority + [P[0][1]], F),
               ([net.clients[o] for o in range(maj)], F), ([net.admins[o] for o in range(maj)], F),
               ([net.orderers[o] for o in range(maj)], F)]
        out.append(("stock_majority_%d_orgs" % n, n, [tree], principals, True, None, [(e, None, c) for e, c in txs]))
    net = network(4)
    P, C = net.org_peers, net.clients                      # C[o] is a client of org o
    org = lambda o: "Org%dMSP" % (o + 1)
    one = lambda p: ([n_of(1, [signed_by(0)])], [p])
    contrast = [([C[0]], None), ([P[0][0]], None)]
    out.append(("role_peer_vs_client", 4, *one(role(org(0), "peer")), True, None, [(e, ns, c) for (e, ns), c in zip(contrast, (F, V))]))
    out.append(("member_principal_accepts_client", 4, [n_of(1, [signed_by(0)])], [org(0)], False, None,
                [(e, ns, c) for (e, ns), c in zip(contrast, (V, V))]))
    out.append(("admin", 4, *one(role(org(0), "admin")), True, None,
                [([net.admins[0]], None, V), ([net.admins_listed[0]], None, V), ([C[0]], None, F), ([P[0][0]], None, F), ([net.admins[1]], None, F),
                 ([net.admins_listed[1]], None, F)]))
    out.append(("orderer", 4, *one(role(org(0), "orderer")), True, None,
                [([net.orderers[0]], None, V), ([P[0][0]], None, F), ([net.admins[0]], None, F), ([net.orderers[1]], None, F)]))
    out.append(("identity", 4, *one(identity_principal(net.peers[0])), True, None,
                [([net.peers[0]], None, V), ([net.peers_alt[0]], None, V), ([P[0][1]], None, F), ([C[0]], None, F), ([net.peers[1]], None, F)]))
    out.append(("member_role_with_bits", 4, *one(role(org(0), "member")), True, None,
                [([C[0]], None, V), ([P[0][1]], None, V), ([net.admins_listed[0]], None, F), ([net.peers[1]], None, F)]))
    wide = [role(org(2 + k % 2), ROLES[k % 5]) for k in range(40)]
    wide[37] = role(org(0), "peer")
    out.append(("principal_in_second_word", 4, [n_of(1, [signed_by(37)])], wide, True, None,
                [([P[0][0]], None, V), ([C[0]], None, F), ([net.orderers[2]], None, F), ([P[2][0]], None, F)]))
    sp, any_tree = stock_endorsement(4, "ANY")
    out.append(("implicit_any", 4, [any_tree], sp, True, None, [([P[2][0]], None, V), ([C[2]], None, F), ([], None, F)]))
    sp, all_tree = stock_endorsement(4, "ALL")
    out.append(("implicit_all", 4, [all_tree], sp, True, None,
                [([P[0][0], P[1][0], P[2][0]], None, F), ([P[0][0], P[1][1], P[2][0], P[3][1]], None, V)]))
    out.append(("implicit_no_sub_policies", 4, [implicit_meta("MAJORITY", [])], sp, True, None,
                [([C[0]], None, V), ([P[0][0]], None, V), ([], None, V)]))
    missing = implicit_meta("MAJORITY", [n_of(1, [signed_by(o)]) for o in range(3)] + [REJECT])
    out.append(("implicit_org_without_sub_policy", 4, [missing], sp, True, None,
                [([P[0][0], P[1][0], P[2][0]], None, V), ([P[0][0], P[1][0], P[3][0]], None, F), ([P[0][0], P[1][0]], None, F)]))
    nested_pr = sp + [role(org(3), "orderer")]
    nested = implicit_meta("ANY", [implicit_meta("MAJORITY", [n_of(1, [signed_by(o)]) for o in range(3)]), implicit_meta("ALL", [n_of(1, [signed_by(4)])])])
    out.append(("implicit_nested_any_of_majority", 4, [nested], nested_pr, True, None,
                [([P[0][0], P[1][0]], None, V), ([P[0][0]], None, F), ([net.orderers[3]], None, V), ([P[3][0]], None, F)]))
    twice = [([P[0][0]], None), ([P[0][0], P[0][1]], None)]
    out.append(("same_role_twice_implicit_all", 4, [implicit_meta("ALL", [n_of(1, [signed_by(0)]), n_of(1, [signed_by(0)])])], [role(org(0), "peer")],
                True, None, [(e, ns, c) for (e, ns), c in zip(twice, (V, V))]))
    out.append(("same_role_twice_n_of_2", 4, [n_of(2, [signed_by(0), signed_by(0)])], [role(org(0), "peer")], True, None,
                [(e, ns, c) for (e, ns), c in zip(twice, (F, V))]))
    both = [(blockgen.CHAINCODE, 1, 1), ("sigcc", 0, 1)]
    sp, maj_tree = stock_endorsement(4)
    out.append(("namespaces_implicit_and_signature_roots", 4, [maj_tree, n_of(2, [signed_by(0), signed_by(3)])], sp, True,
                {blockgen.CHAINCODE: 0, "sigcc": 1},
                [([P[0][0], P[1][0], P[3][0]], both, V), ([P[0][0], P[1][0], P[2][0]], both, F), ([P[0][0], P[1][0], P[2][0]], None, V),
                 ([P[0][0], P[3][0]], both, F)]))
    return out


def materialize(case, seed=61):
    """-> (net, block, info, nodes, principal names, bits or None, {namespace: root} or None, expected codes)."""
    name, n_orgs, trees, principals, use_bits, policies, txs = case
    net = network(n_orgs)
    nodes, roots = forest(trees)
    names = [principal_name(p) for p in principals] if use_bits else list(principals)
    bits = principal_bits(net, principals) if use_bits else None
    pol = {ns: roots[k] for ns, k in policies.items()} if policies else None
    blk, info = blockgen.build_block(net, len(txs), 3, {}, seed=seed, endorsers=lambda t: txs[t][0],
                                     namespaces=lambda t: txs[t][1] or [(blockgen.CHAINCODE, 2, 2)])
    return net, blk, info, nodes, names, bits, pol, [c for _, _, c in txs]
