"""Host model of b2_votes_group_dev (include/b200pos.h, csrc/votes.cuh): every committee's positions stable-sorted by local vote id,
non-attesters (0xFFFFFFFF, or an id outside the committee's range) last in the segment of the committee's last vote.  An independent
restatement of the layout in numpy, for well-formed inputs (no device guard fires)."""
import types

import numpy as np

NONE = 0xFFFFFFFF
INFINITY96 = np.frombuffer(bytes([0xC0]) + bytes(95), dtype=np.uint8)


def group(off, vote, vote_off):
    """(order, seg): order[p] = the committee slot grouped slot p came from; seg = the vote segments, uint[n_votes + 1]"""
    off, vote_off = np.asarray(off, dtype=np.int64), np.asarray(vote_off, dtype=np.int64)
    n_c, n_votes = off.shape[0] - 1, int(vote_off[-1])
    order, seg = np.zeros(int(off[-1]), dtype=np.int64), np.zeros(n_votes + 1, dtype=np.int64)
    for c in range(n_c):
        o0, o1, v0, v1 = int(off[c]), int(off[c + 1]), int(vote_off[c]), int(vote_off[c + 1])
        local = np.asarray(vote[o0:o1]).astype(np.int64)
        key = np.where((local >= v0) & (local < v1), local - v0, v1 - v0)
        p = np.argsort(key, kind="stable")
        order[o0:o1] = o0 + p
        seg[v0:v1] = o0 + np.searchsorted(key[p], np.arange(v1 - v0))
    seg[n_votes] = off[n_c]
    return order, seg


def group_outputs(members, off, vote, vote_off, sigs, bits_stride, c_begin, c_end):
    """Every output of b2_votes_group_dev: members_out, pos_out, seg_off, seg_off_loc (the votes of [c_begin, c_end), over their own
    signatures), bits (prefix rows), agg_bits (aggregation_bits over committee positions) and sigs_out (the range's signatures grouped;
    sigs = the range's own, index 0 = off[c_begin])."""
    off, vote_off = np.asarray(off, dtype=np.int64), np.asarray(vote_off, dtype=np.int64)
    vote = np.asarray(vote).astype(np.int64)
    order, seg = group(off, vote, vote_off)
    n_c, n_votes = off.shape[0] - 1, int(vote_off[-1])
    com = np.repeat(np.arange(n_c), np.diff(off))                     # the committee of every slot
    pos = np.arange(int(off[-1])) - off[com]                          # its position in the committee
    attests = (vote >= vote_off[com]) & (vote < vote_off[com + 1])
    bits = np.zeros((n_votes, 8 * bits_stride), dtype=np.uint8)
    count = np.bincount(vote[attests], minlength=n_votes)
    bits[np.arange(8 * bits_stride)[None, :] < count[:, None]] = 1
    agg = np.zeros((n_votes, 8 * bits_stride), dtype=np.uint8)
    agg[vote[attests], pos[attests]] = 1
    b0, b1 = int(off[c_begin]), int(off[c_end])
    src = np.asarray(sigs, dtype=np.uint8).reshape(-1, 96)
    grouped = order[b0:b1]
    sigs_out = np.where(attests[grouped][:, None], src[grouped - b0], INFINITY96[None, :])
    v0, v1 = int(vote_off[c_begin]), int(vote_off[c_end])
    return types.SimpleNamespace(members_out=np.asarray(members)[order], pos_out=pos[order], seg_off=seg, seg_off_loc=seg[v0:v1 + 1] - b0,
                                 bits=np.packbits(bits, axis=1, bitorder="little"), agg_bits=np.packbits(agg, axis=1, bitorder="little"),
                                 sigs_out=sigs_out.astype(np.uint8))
