"""Oracles of identity admission (fabgpu_msp_identities_add) and of the unknown-identity listing (fabgpu_block_unknown_identities).

listing(envs, known): what the device lists for a block of well-formed envelopes -- for each transaction in order, the serialized
identities it looks up in the MSP table (the creator when the envelope carries a signature, then every endorser whose endorsement
carries signature bytes, in endorsement order) that `known` does not hold, each identity once, at its first appearance.

flags(blk, identities, known_before, ...): the sequence oracle -- block j is validated by oracle/blockval with `known` = the configured
identities plus every identity admitted before block j was submitted."""
from oracle import blockval as ob
from tools import fabricpb as pb


def lookups(env: bytes):
    """The identities one envelope asks the table for, in job order: [creator?] + endorsers.  None when an outer message does not parse."""
    try:
        e = pb.parse(env, {1: ("payload", "bytes"), 2: ("signature", "bytes")})
        p = pb.parse(e["payload"] or b"", {1: ("header", "bytes"), 2: ("data", "bytes")})
        h = pb.parse(p["header"] or b"", {1: ("chdr", "bytes"), 2: ("shdr", "bytes")})
        sh = pb.parse(h["shdr"] or b"", {1: ("creator", "bytes"), 2: ("nonce", "bytes")})
        out = [bytes(sh["creator"])] if e["signature"] and e["payload"] else []
        tx = pb.parse(p["data"] or b"", {1: ("actions", "rep_bytes")})
        ta = pb.parse(tx["actions"][0], {1: ("header", "bytes"), 2: ("payload", "bytes")})
        cap = pb.parse(ta["payload"] or b"", {1: ("cpp", "bytes"), 2: ("action", "bytes")})
        act = pb.parse(cap["action"] or b"", {1: ("prp", "bytes"), 2: ("ends", "rep_bytes")})
        for en in act["ends"]:
            x = pb.parse(en, {1: ("endorser", "bytes"), 2: ("signature", "bytes")})
            if x["signature"]:
                out.append(bytes(x["endorser"] or b""))
        return out
    except (pb.PbError, IndexError, TypeError):
        return None


def listing(envs, known):
    """[(serialized, first tx)] of the identities the block looks up and `known` does not hold, distinct, in first-appearance order"""
    known = {bytes(k) for k in known}
    seen, out = set(), []
    for t, env in enumerate(envs):
        for ser in lookups(env) or []:
            if ser in known or ser in seen:
                continue
            seen.add(ser)
            out.append((ser, t))
    return out


def envelopes(info):
    blob, off = info["env_blob"], info["env_off"]
    return [bytes(blob[off[t]:off[t + 1]]) for t in range(len(off) - 1)]


def flags(blk, identities, known, channel, nodes, principals, policies=None):
    """The flags of one block with the device table holding `known` (the configured and the admitted identities' serialized bytes)
    and `identities` every identity the oracle's MSP can deserialise (configured and to be admitted)"""
    return ob.validate_block(blk, identities, channel, nodes, principals, policies=policies, known=list(known))
