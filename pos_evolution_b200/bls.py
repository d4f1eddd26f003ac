"""The ``bls`` facade of the executable consensus spec (eth2spec.utils.bls), served by the H100.

Same names, argument meaning and error behaviour as the module the reference calls
(pos-evolution.md:165 ``bls.Verify``; BASELINE.json names ``bls.Aggregate`` and
``bls.FastAggregateVerify``): verification functions never raise and return False for any
malformed input; ``Aggregate`` raises ValueError on an empty list or an undecodable signature, ``AggregatePKs`` on an empty list or
a key that fails KeyValidate.  The Altair helpers ``eth_fast_aggregate_verify`` and ``eth_aggregate_pubkeys`` (what
process_sync_aggregate calls) are here too; the second raises AssertionError, as upstream.
Every call goes through the C ABI (include/b200pos.h) to hand-written sm_90a kernels; there is
no CPU path.  These per-call functions move a few hundred bytes over PCIe each -- for throughput
use the batch API (pos_evolution_b200.engine.Engine / spec.EpochProcessor).

Messages are 32-byte SSZ signing roots (the only thing pyspec ever signs): other lengths raise
ValueError, a contract violation rather than an invalid signature.
"""
from typing import Sequence

import numpy as np

from .engine import Engine

_engine = None


def use_engine(engine: Engine):
    """Route the module-level functions through an existing Engine (one per process/GPU)."""
    global _engine
    _engine = engine


def engine() -> Engine:
    global _engine
    if _engine is None:
        _engine = Engine(0)
    return _engine


R_ORDER = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001


def _msg(message) -> bytes:
    m = bytes(message)
    if len(m) != 32:
        raise ValueError("message must be a 32-byte signing root")
    return m


def SkToPk(privkey: int) -> bytes:
    if not 0 < int(privkey) < R_ORDER:
        raise ValueError("secret key out of range")
    return bytes(engine().sk_to_pk([int(privkey)])[0])


def Sign(privkey: int, message: bytes) -> bytes:
    if not 0 < int(privkey) < R_ORDER:
        raise ValueError("secret key out of range")
    m = np.frombuffer(_msg(message), dtype=np.uint8).reshape(1, 32)
    return bytes(engine().sign([int(privkey)], [0], m)[0])


def FastAggregateVerify(pubkeys: Sequence[bytes], message: bytes, signature: bytes) -> bool:
    m = _msg(message)
    try:
        pks = [bytes(p) for p in pubkeys]
        sig = bytes(signature)
        if len(pks) < 1 or len(sig) != 96 or any(len(p) != 48 for p in pks):
            return False
        ok = engine().fast_aggregate_verify_pks(np.frombuffer(b"".join(pks), dtype=np.uint8), [0, len(pks)],
                                                np.frombuffer(m, dtype=np.uint8), np.frombuffer(sig, dtype=np.uint8))
        return bool(ok[0])
    except (TypeError, ValueError):
        return False


def Verify(PK: bytes, message: bytes, signature: bytes) -> bool:
    return FastAggregateVerify([PK], message, signature)


def AggregateVerify(pubkeys: Sequence[bytes], messages: Sequence[bytes], signature: bytes) -> bool:
    """One signature over (pubkeys[i], messages[i]) pairs; messages need not be distinct (proof-of-possession scheme)."""
    try:
        msgs = list(messages)
    except TypeError:
        return False
    ms = [_msg(m) for m in msgs]
    try:
        pks = [bytes(p) for p in pubkeys]
        sig = bytes(signature)
        if len(pks) < 1 or len(pks) != len(ms) or len(sig) != 96 or any(len(p) != 48 for p in pks):
            return False
        ok = engine().aggregate_verify_pks(np.frombuffer(b"".join(pks), dtype=np.uint8), [0, len(pks)],
                                           np.frombuffer(b"".join(ms), dtype=np.uint8), np.frombuffer(sig, dtype=np.uint8))
        return bool(ok[0])
    except (TypeError, ValueError):
        return False


B2_PK_INVALID_KEY, B2_PK_EMPTY = 1, 2


def AggregatePKs(pubkeys: Sequence[bytes]) -> bytes:
    """Sum of the keys, compressed (the infinity encoding when they cancel); ValueError on an empty list or a key that fails
    KeyValidate."""
    pks = [bytes(p) for p in pubkeys]
    if len(pks) < 1:
        raise ValueError("AggregatePKs: empty list")
    if any(len(p) != 48 for p in pks):
        raise ValueError("AggregatePKs: key is not 48 bytes")
    out, status = engine().aggregate_pks(np.frombuffer(b"".join(pks), dtype=np.uint8), [0, len(pks)])
    if status[0] & (B2_PK_INVALID_KEY | B2_PK_EMPTY):
        raise ValueError("AggregatePKs: invalid key")
    return bytes(out[0])


_AggregatePKs = AggregatePKs          # the name pyspec's wrapper calls on its backend


def KeyValidate(pubkey: bytes) -> bool:
    """decodable, not infinity, in G1 (b2_key_validate: the registry loader's kernel on a scratch buffer; the shared engine's
    registry is left alone)."""
    pk = bytes(pubkey)
    if len(pk) != 48:
        return False
    return bool(engine().key_validate(np.frombuffer(pk, dtype=np.uint8))[0])


def Aggregate(signatures: Sequence[bytes]) -> bytes:
    sigs = [bytes(s) for s in signatures]
    if len(sigs) < 1:
        raise ValueError("Aggregate: empty list")
    if any(len(s) != 96 for s in sigs):
        raise ValueError("Aggregate: signature is not 96 bytes")
    out, status = engine().aggregate(np.frombuffer(b"".join(sigs), dtype=np.uint8), [0, len(sigs)])
    if status[0] != 0:
        raise ValueError("Aggregate: undecodable signature")
    return bytes(out[0])


def AggregateBatch(signatures96: np.ndarray, seg_off):
    """Batched bls.Aggregate: segment s = rows [seg_off[s], seg_off[s+1]).  -> (uint8[n_seg,96], int32[n_seg] status)."""
    return engine().aggregate(signatures96, seg_off)


# ---- Altair bls helpers (restated from the upstream consensus specs, specs/altair/bls.md; not part of the reference's text)
G2_POINT_AT_INFINITY = bytes([0xC0]) + bytes(95)


def eth_aggregate_pubkeys(pubkeys: Sequence[bytes]) -> bytes:
    """Sum of the keys, compressed; AssertionError on an empty list or a key that fails KeyValidate."""
    pks = [bytes(p) for p in pubkeys]
    assert len(pks) > 0, "eth_aggregate_pubkeys: empty list"
    assert all(len(p) == 48 for p in pks), "eth_aggregate_pubkeys: key is not 48 bytes"
    out, status = engine().aggregate_pks(np.frombuffer(b"".join(pks), dtype=np.uint8), [0, len(pks)])
    assert not status[0] & (B2_PK_INVALID_KEY | B2_PK_EMPTY), "eth_aggregate_pubkeys: invalid key"
    return bytes(out[0])


def eth_fast_aggregate_verify(pubkeys: Sequence[bytes], message: bytes, signature: bytes) -> bool:
    """FastAggregateVerify, except that an empty key list verifies exactly the G2 infinity signature."""
    try:
        if len(pubkeys) == 0 and bytes(signature) == G2_POINT_AT_INFINITY:
            return True
    except TypeError:
        return False
    return FastAggregateVerify(pubkeys, message, signature)
