"""ORACLE extension (test infrastructure, NOT product code): the committed tx-id check over every block oracle of the suite.

  checkTxIdDupsLedger     core/committer/txvalidator/v20/validator.go:363-372,462-491 (v14/validator.go:334-345,450ff, same place):
                          after ValidateTransaction and the channel check (TARGET_CHAIN_NOT_FOUND), before the dispatcher / VSCC, every
                          endorser transaction's id is looked up with GetTransactionByID (core/ledger/kvledger/kv_ledger.go:362-375):
                            found                 -> DUPLICATE_TXID (9)
                            NotFoundInIndexErr    -> on to the dispatcher
                            any other error       -> a terminal error of the block; the device hands the transaction to the CPU (254).
                                                     An id imported from a snapshot (empty index value, blockindex.go:244-246) is one.
  Config transactions never reach it.  A transaction that does has passed CheckTxID, so only canonical ids can match; the table maps
  the id string to its kind (0: found, 1: the lookup fails), exactly as fabgpu_committed_txids takes it.

Every oracle here calls oracle.blockval.validate_tx first, and decides nothing about a transaction that validate_tx does not return
VALID for.  `committed(oracle_fn, ...)` runs one of them with validate_tx answering 9 / 254 at the ledger check's place for the ids of
the table: a transaction that reaches the channel check and passes it, whose id the table holds.  The in-block duplicate pass, the
key-level dependency rule and the v1.3 lscc pass then see those codes as they see any other failure of the transaction.
"""
import contextlib

from oracle import blockval as ob
from tools import fabricpb as pb


def txid_of(env_bytes):
    """ChannelHeader.tx_id of an envelope, or None where it does not parse"""
    try:
        env = pb.parse(env_bytes, ob.S_ENVELOPE)
        hdr = pb.parse(pb.parse(env["payload"] or b"", ob.S_PAYLOAD)["header"] or b"", ob.S_HEADER)
        return (pb.parse(hdr["channel_header"] or b"", ob.S_CHDR)["tx_id"] or b"").decode("utf-8", "replace")
    except pb.PbError:
        return None


def _plain(msp):
    """the MSP's table without the state a caller's subclass keeps per transaction (v13_oracle's lazy endorser check)"""
    m = ob.Msp.__new__(ob.Msp)
    m.by_bytes, m.known = msp.by_bytes, msp.known
    return m


@contextlib.contextmanager
def ledger(table):
    """oracle.blockval.validate_tx with the ledger check, for the duration of the block; table: {tx id str: kind 0 / 1}"""
    inner = ob.validate_tx

    def validate_tx(env_bytes, msp, channel, *args, **kw):
        # the checks up to the channel's: with a channel no transaction names, a transaction passing all of them is 14
        if inner(env_bytes, _plain(msp), _NO_CHANNEL, *args, **kw)[0] == ob.TARGET_CHAIN_NOT_FOUND:
            env = pb.parse(env_bytes, ob.S_ENVELOPE)
            hdr = pb.parse(pb.parse(env["payload"], ob.S_PAYLOAD)["header"], ob.S_HEADER)
            chdr = pb.parse(hdr["channel_header"] or b"", ob.S_CHDR)
            txid = (chdr["tx_id"] or b"").decode("utf-8", "replace")
            if (chdr["channel_id"] or b"").decode("utf-8", "replace") == channel and txid in table:
                return (ob.DUPLICATE_TXID if table[txid] == 0 else ob.NOT_VALIDATED), ""
        return inner(env_bytes, msp, channel, *args, **kw)

    ob.validate_tx = validate_tx
    try:
        yield
    finally:
        ob.validate_tx = inner


class _Never:
    """a channel name equal to no decoded channel id"""

    def __eq__(self, other):
        return False

    def __ne__(self, other):
        return True


_NO_CHANNEL = _Never()


def committed(oracle_fn, *args, committed=None, **kw):
    """oracle_fn(*args, **kw) -- any block oracle of the suite -- with the committed tx-id table `committed` ({id str: kind}); None = no
    table installed, which is oracle_fn itself.  The table may hold any strings: a non-canonical one never equals a transaction's id
    that passed CheckTxID."""
    if committed is None:
        return oracle_fn(*args, **kw)
    with ledger(dict(committed)):
        return oracle_fn(*args, **kw)
