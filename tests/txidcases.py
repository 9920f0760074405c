"""Test infrastructure (not product code): the committed tx-id cases (fabgpu_committed_txids: checkTxIdDupsLedger on the device) that the
oracle, the host build and the device are all held to, with every expected code written out.

The channel, node array, principals, namespace table and lscc versions are v13cases' (mycc wants 2 of 4 orgs, othercc 1 of 4, ghostcc has
no entry); each endorsing org signs with its first peer.  Each transaction says what the ledger holds for its ChannelHeader.tx_id:
  None       nothing
  0 / 1      its id with kind 0 (committed) / 1 (GetTransactionByID fails)
  "0then1"   its id with kind 0 in the replacing call and kind 1 in a later _add
  "upper", "short", "long"    its id upper-cased, without its last character, with one more: never canonical, never a match
"""
from oracle import blockval as ob
import klcases
import txid_oracle
import v13_oracle
import v13cases

V, F, NV, DUP = ob.VALID, ob.ENDORSEMENT_POLICY_FAILURE, ob.NOT_VALIDATED, ob.DUPLICATE_TXID
CC, OTHER, GHOST = v13cases.CC, v13cases.OTHER, v13cases.GHOST
MODE_V20, MODE_V13 = 0, 1
policies, versions = v13cases.policies, v13cases.versions


def tx(orgs, namespaces, code, ledger=None, cc=(CC, "1.0"), fault=None):
    return (orgs, namespaces, fault, code, cc, ledger)


def cases():
    """[(name, mode, key table: True = klcases' filler table, else none, [tx(...)])]"""
    pub = [(CC, 1, 1)]
    return [
        ("committed_is_duplicate", MODE_V20, False, [tx([0, 1], pub, DUP, 0), tx([0, 1], pub, V)]),
        ("unanswerable_is_not_validated", MODE_V20, False, [tx([0, 1], pub, NV, 1), tx([0, 1], pub, V)]),
        # checks before the ledger's keep their codes
        ("earlier_codes_win", MODE_V20, False,
         [tx([0, 1], pub, ob.BAD_CREATOR_SIGNATURE, 0, fault="bad_creator_sig"), tx([0, 1], pub, ob.BAD_PROPOSAL_TXID, 0, fault="bad_txid"),
          tx([0, 1], pub, ob.INVALID_ENDORSER_TRANSACTION, 0, fault="bad_proposal_hash"),
          tx([0, 1], pub, ob.TARGET_CHAIN_NOT_FOUND, 0, fault="wrong_channel"),
          tx([0, 1], pub, ob.UNSUPPORTED_TX_PAYLOAD, 0, fault="config_update_type"), tx([0, 1], pub, NV, 0, fault="unknown_creator"),
          tx([0, 1], pub, V)]),
        # and those after it lose
        ("later_codes_lose", MODE_V20, False,
         [tx([0, 1], pub, DUP, 0, fault="cc_name_mismatch"), tx([0, 1], pub, DUP, 0, fault="dup_namespace"),
          tx([0, 1], [(GHOST, 1, 1)], DUP, 0, cc=(GHOST, "1.0")), tx([0, 1], pub, DUP, 0, fault="unknown_endorser"), tx([0], pub, DUP, 0),
          tx([0, 1], pub, DUP, 0, fault="bad_header_extension"), tx([0, 1], [(GHOST, 1, 1)], NV, cc=(GHOST, "1.0")), tx([0, 1], pub, V)]),
        ("ledger_and_in_block_duplicates", MODE_V20, False,
         [tx([0, 1], pub, DUP, 0), tx([0, 1], pub, DUP, fault="dup_txid"), tx([0, 1], pub, V), tx([0, 1], pub, DUP, fault="dup_txid"),
          tx([0, 1], pub, NV, 1), tx([0, 1], pub, NV, fault="dup_txid")]),
        # a ledger duplicate never reaches VSCC: a later writer of a key it metadata-writes would wait forever
        ("duplicate_metadata_writer", MODE_V20, True,
         [tx([0, 1], [klcases.pub(md=["d1"])], DUP, 0), tx([0, 1], [klcases.pub("d1")], NV), tx([0, 1], [klcases.pub(md=["d2"])], V),
          tx([0, 1], [klcases.pub("d2")], F)]),
        ("v13_duplicate_lscc_invocation", MODE_V13, False,
         [tx([0, 1], [("lscc", 0, 1)], DUP, 0, cc=("lscc", "1.0")), tx([0, 1], pub, V), tx([0], pub, F), tx([0, 1], pub, DUP, 0),
          tx([0, 1], pub, v13_oracle.EXPIRED_CHAINCODE, cc=(CC, "2.0")), tx([0, 1], pub, DUP, 0, cc=(CC, "2.0"))]),
        ("v13_unanswerable_lscc_invocation_marks_the_block", MODE_V13, False,
         [tx([0, 1], [("lscc", 0, 1)], NV, 1, cc=("lscc", "1.0")), tx([0, 1], pub, NV), tx([0], pub, F)]),
        ("non_canonical_ids_never_match", MODE_V20, False,
         [tx([0, 1], pub, V, "upper"), tx([0, 1], pub, V, "short"), tx([0, 1], pub, V, "long"), tx([0, 1], pub, DUP, 0)]),
        ("kind_raised_by_a_later_add", MODE_V20, False, [tx([0, 1], pub, NV, "0then1"), tx([0, 1], pub, DUP, 0)]),
    ]


def materialize(case, seed=149):
    """-> (net, block, info, codes, set calls [(replace, ids, kinds)], the oracle's table {id: kind})"""
    import nodeou
    from tools import blockgen
    txs = case[3]
    net = nodeou.network(4)
    faults = {t: x[2] for t, x in enumerate(txs) if x[2]}
    blk, info = blockgen.build_block(net, len(txs), 3, faults, seed=seed, endorsers=lambda t: [net.org_peers[o][0] for o in txs[t][0]],
                                     namespaces=lambda t: txs[t][1], chaincode=lambda t: txs[t][4])
    envs = [bytes(info["env_blob"][info["env_off"][t]:info["env_off"][t + 1]]) for t in range(len(txs))]
    ids = [txid_oracle.txid_of(e) for e in envs]
    first, later = ([], []), ([], [])
    for t, x in enumerate(txs):
        led, i = x[5], ids[t]
        if led in (0, 1):
            first[0].append(i); first[1].append(led)
        elif led == "0then1":
            first[0].append(i); first[1].append(0); later[0].append(i); later[1].append(1)
        elif led == "upper":
            first[0].append(i.upper()); first[1].append(0)
        elif led == "short":
            first[0].append(i[:-1]); first[1].append(0)
        elif led == "long":
            first[0].append(i + "0"); first[1].append(0)
    first[0].append(""); first[1].append(0)                  # an empty id: never a match
    calls = [(True, first[0], first[1])] + ([(False, later[0], later[1])] if later[0] else [])
    table = {}
    for _, cids, kinds in calls:
        for i, k in zip(cids, kinds):
            table[i] = max(table.get(i, 0), k)
    return net, blk, info, [x[3] for x in txs], calls, table


def oracle_flags(case, blk, net, names, bits, table, collections=None):
    """the oracle of the case's mode, with the committed table"""
    ids = net.identities()
    kt = klcases.key_table((case[0], False, {}, case[3])) if case[2] else None
    nodes, vps = klcases.combined(*kt) if kt else (v13cases.collcases.forest()[0], None)
    if case[1] == MODE_V13:
        return txid_oracle.committed(v13_oracle.validate_block, blk, ids, net.channel, nodes, names, bits=bits, policies=policies(),
                                     versions=versions(), collections=collections, vps=vps, known=[i[0] for i in ids], committed=table)
    import keylevel_oracle
    return txid_oracle.committed(keylevel_oracle.validate_block, blk, ids, net.channel, nodes, names, bits=bits, policies=policies(),
                                 collections=collections, vps=vps, known=[i[0] for i in ids], committed=table)
