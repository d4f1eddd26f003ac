"""EpochProcessor -- the batch (array-level) public API for one rank / one GPU.

One call processes a whole epoch of attestations:
  individual G2 signatures --bls.Aggregate per committee--> aggregate signatures
  --FastAggregateVerify (registry-indexed pubkey gather + hash-to-G2 + pairing)--> verdicts
  --update_latest_messages (accepted aggregates only)--> LMD table on the device
  --get_weight scatter--> per-block direct votes  [--NCCL all-reduce over ranks--]  --get_head--> head index.
(pos-evolution.md:722-754, :963-979, :1102-1116, :1435-1441.)

Two ways to drive it:
  * `process_epoch_dev` / `process_epoch_host`: synchronous in stream order, one epoch at a time;
  * `submit_dev` / `submit_host` + `drain`: software-pipelined over `depth` slots (default 3, at most B2_EPOCH_SLOTS = 16).
    The signature decompression of epoch k+1 (grid-filling, integer-pipe bound) overlaps with the latency-bound tails of
    the epochs before it (subgroup check, second Miller loop, final exponentiation, LMD update; each on its slot's own
    high-priority streams inside the library) and with their fork choice (on this object's fork-choice stream); in the
    host form the H2D copy of epoch k+1 overlaps too.  `submit_*` returns the ticket of the epoch submitted depth-1
    calls earlier.
The synchronous forms and `get_head` use slot 0 and the one vote accumulator of the pipeline, so they need it drained: while
submitted epochs are in flight (until `drain()` has returned) they raise AssertionError before enqueueing anything.

Multi-GPU, two layouts (SURVEY.md section 8e):
  * `shard=None` (weak scaling): every rank owns its OWN validator set and epoch; the only exchange is the u64[n_blocks]
    all-reduce of direct vote weights (int64 two's-complement sum == u64 sum) between the vote scatter and get_head.
  * `shard=(rank, world)` (strong scaling -- BASELINE.json configs 4/5): ONE validator set and ONE epoch for the whole
    box.  Committees are disjoint within an epoch (pos-evolution.md:455, :472-474), so rank g aggregates and verifies the
    aggregates [g*n_agg/world, (g+1)*n_agg/world) -- its slots -- from ITS slice of the individual signatures, against a
    replicated registry.  Exchange per epoch: one all-gather of (aggregate signature 96 B + verdict 1 B) per aggregate,
    after which EVERY rank applies update_latest_messages for ALL accepted aggregates to its replica of the LMD table
    (12 B per set bit, microseconds); then get_head: rank g scatters the votes of validators [g*N/world, (g+1)*N/world)
    only, one u64[n_blocks] all-reduce, head on every rank.  No collective touches the BLS data path.

Slashing detection (`enable_slasher`): after each epoch's fork choice, on the fork-choice stream and so in epoch order, the slasher
(include/b200pos.h, b2_slasher_*) records and checks every accepted aggregate of the epoch; `Ticket.slashings()` reports the flagged
member slots.  Sharded, rank g holds the history of validators [g*N/world, (g+1)*N/world) only -- the range of its vote scatter --
and reports those; the ranks' reports together are the unsharded one, with no collective added.

Vote form (`EpochProcessor(..., max_votes=M)` and `votes=(vote, vote_off)` on any entry point): the members of one committee may sign
different AttestationData (a late block, a fork: pos-evolution.md:1321-1348).  vote u32[n_sig] names the vote id each member signed
(0xFFFFFFFF: did not attest), the ids of committee c are [vote_off[c], vote_off[c+1]) (strictly increasing; n_votes = vote_off[-1] <=
M), and msgs / target epochs / block indices / source epochs are per vote.  The device groups the epoch by vote (Engine.votes_group_dev,
on the stream that claimed the slot) and the epoch kernels run unchanged with one aggregate per vote; Ticket.wait() /
aggregate_signatures() / aggregation_bits() then hold one row per vote, i.e. one Attestation each.  Sharded, rank g aggregates the votes
of its committees [vote_off[c0_g], vote_off[c1_g]); the all-gather pads every rank's block to the largest count.

Attestation intake (`intake_dev`): an epoch of unaggregated Attestations straight off the wire is checked against the device tree
(process_attestation, validate_on_attestation), one kept per committee position, and turned into the vote form's inputs on the device
(Engine.attestation_intake_dev); the returned tensors go to submit_dev / process_epoch_dev with votes=(r.vote, r.vote_off).
`intake_single_dev` does the same for Electra's SingleAttestations (Engine.single_attestation_intake_dev).

Equivocation discounting (`enable_slasher(..., discount=True)`, pos-evolution.md:1405-1461): right after each epoch's slasher update,
every validator it flagged joins the device's Store.equivocating_indices, so from the next epoch on its votes neither move its latest
message nor count in a head (:1411: votes of validators "not viewed to have equivocated at previous slots").  The marks only grow.
Sharded, rank g marks its own range; each rank's slice of the table is then all-gathered and merged into every replica, on the
fork-choice stream before the next epoch's exchange, so the replicas of the LMD table stay identical.
"""
import collections
import contextlib

import numpy as np
import torch

from .engine import Engine

MAX_DEPTH = 16      # == B2_EPOCH_SLOTS (include/b200pos.h)


# One epoch's arrays: n aggregates (committees, or votes when `votes`) over members[off[a] .. off[a+1]); this rank's rows [r0, r1) with members_loc /
# off_loc over its own signatures `sigs`; sharded, `pad` rows per rank in the all-gather of out_loc into out_all and, in the vote form,
# `ranges` = (first row, count) of every rank.
_Layout = collections.namedtuple("_Layout", "votes n members off r0 r1 members_loc off_loc sigs pad ranges out_loc out_all")

Intake = collections.namedtuple("Intake", "sigs vote msgs target_epoch block_idx source_epoch data128 status vote_off")
Intake.__doc__ = """One epoch's attestations after EpochProcessor.intake_dev: fresh device tensors sigs uint8[n_sig, 96] (committee order), vote
int32[n_sig], and per vote (min(n_votes, max_votes) rows) msgs uint8[., 32], target_epoch / source_epoch int64, block_idx int32, data128
uint8[., 128];
status int32[n_att] per attestation (include/b200pos.h, b2_attestation_intake); vote_off int64[n_committees + 1] on the host.  Submit
with submit_dev(r.sigs, None, r.msgs, r.target_epoch, r.block_idx, votes=(r.vote, r.vote_off), source_epoch=r.source_epoch)."""

Slashings = collections.namedtuple("Slashings", "status aggregate position validator kind surrounded_target surrounding_target")
Slashings.__doc__ = """What the slasher found in one epoch (numpy arrays).  status: int32[n_agg], B2_SLASHER_* per aggregate.  One entry per
flagged member slot: aggregate index, position in the committee, validator index, kind (B2_SLASHABLE_* bits: 1 double, 2 surrounds,
4 surrounded), the smallest target among the attestations it surrounds and the largest target among those surrounding it
(0xffffffff where that bit is clear).  A conflicting target names the epoch batch that holds the partner attestation."""


class _Slot:
    """Everything one epoch in flight owns (slot i of the pipeline; the synchronous forms use slot 0)."""

    def __init__(self, i, ep):
        z, h, n = ep._zeros, ep._pinned, ep.rows
        self.i = i
        # staged inputs (EpochProcessor._stage); set_committees sizes the signatures, enable_slasher adds the source epochs
        self.sigs = self.src = None
        self.bits, self.msgs = z((n, ep.bits_stride), torch.uint8), z((n, 32), torch.uint8)
        self.tgt, self.blk = z(n, torch.int64), z(n, torch.int32)
        # device outputs
        self.agg_sig, self.agg_status = z((n, 96), torch.uint8), z(max(ep.n_loc, ep.max_votes or 0), torch.int32)
        self.ok, self.head = z(n, torch.uint8), z(1, torch.int32)
        if ep.sharded:
            # this rank's outputs packed for ONE all-gather per epoch: n_loc aggregate signatures, then n_loc verdict bytes
            self.out_loc, self.out_all = z(ep.n_loc * 97, torch.uint8), z((ep.world, ep.n_loc * 97), torch.uint8)
        # pinned host readback
        self.h_ok, self.h_head, self.h_agg_sig = h(n, torch.uint8), h(1, torch.int32), h((n, 96), torch.uint8)
        # pipelined forms: the fork choice (+ D2H) and the slasher update of the epoch that last used the slot
        self.ev_fc = self.ev_sl = None
        self.layout = None                # the epoch's _Layout (EpochProcessor._committee_layout / _group)
        if ep.max_votes:
            # vote form: the epoch grouped by vote (the bit rows go to self.bits); the signatures are sized by set_committees
            mv = ep.max_votes
            self.v_members, self.v_pos, self.v_vote = z(ep.n_sig, torch.int32), z(ep.n_sig, torch.int32), z(ep.n_sig, torch.int32)
            self.v_seg, self.v_seg_loc = z(mv + 1, torch.int32), z(mv + 1, torch.int32)
            self.v_aggbits, self.h_aggbits = z((mv, ep.bits_stride), torch.uint8), h((mv, ep.bits_stride), torch.uint8)
            self.v_vote_off, self.h_vote_off, self.ev_vote_off = z(ep.n_agg + 1, torch.int32), h(ep.n_agg + 1, torch.int32), None
            self.v_sigs = None
            if ep.sharded:                # as out_loc / out_all, padded to the largest rank's vote count
                self.vout_loc, self.vout_all = z(mv * 97, torch.uint8), z(ep.world * mv * 97, torch.uint8)

    def enable_slasher(self, ep, discount):
        z, h = ep._zeros, ep._pinned
        self.src = z(ep.rows, torch.int64)
        self.sl_status, self.sl_kind = z(ep.rows, torch.int32), z(ep.n_sig, torch.uint8)
        self.sl_conflict, self.sl_flagged = z((ep.n_sig, 2), torch.int32), z(1, torch.int32)
        self.h_sl_status, self.h_sl_flagged = h(ep.rows, torch.int32), h(1, torch.int32)
        if discount:      # per member slot: 1 where the discount newly marked its validator; how many
            self.sl_new, self.sl_n_new, self.h_sl_n_new = z(ep.n_sig, torch.uint8), z(1, torch.int32), h(1, torch.int32)


class _Ticket:
    """Result of one submitted epoch: verdict bytes + head index (+ the aggregate signatures), valid after .wait() and until
    `depth` further epochs have been submitted; with the slasher on, also its findings (.slashings())."""

    def __init__(self, ep, slot, host):
        self._ep, self._slot, self._host = ep, slot, host
        self.slot = slot.i                                # the pipeline slot the epoch ran in (EpochProcessor.d_agg_status[slot])
        self.n, self.votes = slot.layout.n, slot.layout.votes
        self.d_agg_sig, self.event, self.slasher_event = slot.agg_sig[:self.n], slot.ev_fc, slot.ev_sl

    def wait(self):
        """(verdict bytes, head index): one verdict per committee, or per vote in the vote form"""
        self.event.synchronize()
        if self._host:
            return self._slot.h_ok[:self.n].clone(), int(self._slot.h_head[0])
        return self._slot.ok[:self.n], int(self._slot.head[0])

    def aggregate_signatures(self):
        """bls.Aggregate's result for every committee (vote) of the epoch (uint8[n, 96]; 96 zero bytes where nobody signed); host tensor
        in the host form."""
        self.event.synchronize()
        return self._slot.h_agg_sig[:self.n].clone() if self._host else self.d_agg_sig

    def aggregation_bits(self):
        """Vote form: every vote's aggregation_bits over its committee's positions (uint8[n_votes, bits_stride], SSZ Bitlist order without
        the delimiter); host tensor in the host form."""
        assert self.votes, "aggregation_bits: the epoch was not submitted in the vote form"
        self.event.synchronize()
        return self._slot.h_aggbits[:self.n].clone() if self._host else self._slot.v_aggbits[:self.n]

    def slashings(self) -> Slashings:
        """The slasher's findings for this epoch (waits for its update, which runs after the head); EpochProcessor.enable_slasher first."""
        assert self.slasher_event is not None, "no slasher: EpochProcessor.enable_slasher"
        return self._ep._read_slashings(self._slot, self._host, self.slasher_event)

    def n_flagged(self) -> int:
        """Only the number of flagged member slots of this epoch (waits for the slasher's update; no kind or conflict copy)."""
        assert self.slasher_event is not None, "no slasher: EpochProcessor.enable_slasher"
        self.slasher_event.synchronize()
        return int((self._slot.h_sl_flagged if self._host else self._slot.sl_flagged)[0])

    def discounted(self):
        """The validators this epoch's discount newly marked as equivocating, sorted (int64 numpy array; waits for the slasher's update);
        enable_slasher(..., discount=True) first."""
        assert self.slasher_event is not None and self._ep.discount, "no discount: EpochProcessor.enable_slasher(..., discount=True)"
        return self._ep._read_discounted(self._slot, self._host, self.slasher_event)


class EpochProcessor:
    def __init__(self, engine: Engine, n_agg: int, n_sig: int, bits_stride: int, n_blocks: int, process_group=None, device=None, depth: int = 3,
                 shard=None, n_validators=None, tail_form: str = "auto", max_votes: int = None):
        """n_agg / n_sig: aggregates and individual signatures of the WHOLE epoch (in sharded mode this rank handles 1/world of
        them).  tail_form: "thread" (fewest instructions and smallest footprint; needs depth x step > the ~30-40 ms a tail lasts),
        "team" (three lanes per pairing: shortest critical path) or "auto" (= thread: measured best at 1, 2, 4 and 8 GPUs, see
        DESIGN.md section 6b).  Independently of it the last `team_last` epochs of a batch take the team form (drain_hint).
        max_votes: capacity of the vote form (votes= on the entry points; the module docstring); every slot then owns the grouped
        buffers and per-vote outputs of up to max_votes votes.  None: no vote form, nothing allocated for it."""
        self.eng = engine
        self.dev = device if device is not None else torch.device("cuda", engine.device)
        self.pg = process_group
        self.n_agg, self.n_sig, self.n_blocks, self.bits_stride = n_agg, n_sig, n_blocks, bits_stride
        assert max_votes is None or int(max_votes) > 0, "max_votes: a positive capacity, or None"
        self.max_votes = None if max_votes is None else int(max_votes)
        self.rows = n_agg if max_votes is None else max(n_agg, self.max_votes)      # rows of the per-aggregate slot buffers
        cuda = self.dev.type == "cuda"
        assert 2 <= depth <= MAX_DEPTH, "depth must be 2..B2_EPOCH_SLOTS"
        self.depth = depth
        if shard is not None:
            self.rank, self.world = int(shard[0]), int(shard[1])
            assert 0 <= self.rank < self.world and n_agg % self.world == 0, "aggregates must divide evenly over the ranks"
            assert n_validators is not None, "sharded epochs need the size of the (replicated) registry"
        else:
            self.rank, self.world = 0, 1
        self.sharded = shard is not None and self.world > 1
        self.n_val = n_validators
        self.a0, self.a1 = self.rank * n_agg // self.world, (self.rank + 1) * n_agg // self.world
        self.n_loc = self.a1 - self.a0
        if self.sharded:
            self.v0, self.v1 = self.rank * n_validators // self.world, (self.rank + 1) * n_validators // self.world
        self.d_votes = self._zeros(n_blocks, torch.int64)
        self.n_sig_loc = None        # set by set_committees
        self.slots = [_Slot(i, self) for i in range(depth)]
        # each slot's aggregate signatures and bls.Aggregate statuses, indexed by slot (Ticket.slot); the slots' own tensors
        self.d_agg_sig = [s.agg_sig for s in self.slots]
        self.h_agg_sig = [s.h_agg_sig for s in self.slots]
        self.d_agg_status = [s.agg_status for s in self.slots]
        self.copy_stream = torch.cuda.Stream(device=self.dev) if cuda else None
        self.fc_stream = torch.cuda.Stream(device=self.dev) if cuda else None
        self.k = 0
        self._inflight = collections.deque()      # tickets of the submitted, not yet returned epochs
        self._team_form = False
        assert tail_form in ("auto", "thread", "team")
        # Measured on 2 and 8 GPUs of an earlier generation (not re-measured on H100s): the thread-per-aggregate tail wins at every N as long as enough epochs are
        # in flight to cover its latency (N = 2: 18.5 ms thread / depth 4 against 21.7 ms team; N = 8: 6.32 against 6.80) -- the one-warp
        # team blocks with their 49 KB of shared memory displace more decompression blocks than their shorter latency is worth.
        self.always_team = tail_form == "team"
        # ... except at the end of a batch: the last `team_last` epochs take the team form (see drain_hint)
        self.team_last = 1
        self.slasher = False          # enable_slasher
        self.discount = False

    def _zeros(self, shape, dtype):
        return torch.zeros(shape, dtype=dtype, device=self.dev)

    def _pinned(self, shape, dtype):
        return torch.zeros(shape, dtype=dtype, pin_memory=self.dev.type == "cuda")

    def set_committees(self, members, off):
        """members u32[n_sig] (committee order), off u32[n_agg+1] for the WHOLE epoch; signature j belongs to member j."""
        off64 = off.astype("int64")
        self.d_members = torch.as_tensor(members.astype("int32"), device=self.dev)
        self.d_off = torch.as_tensor(off.astype("int32"), device=self.dev)
        self.m0, self.m1 = int(off64[self.a0]), int(off64[self.a1])
        self.n_sig_loc = self.m1 - self.m0
        # this rank's rows: members of its aggregates and offsets relative to its first member
        self.d_members_loc = self.d_members[self.m0:self.m1]
        self.d_off_loc = torch.as_tensor((off64[self.a0:self.a1 + 1] - off64[self.a0]).astype("int32"), device=self.dev)
        for s in self.slots:
            s.sigs = self._zeros((self.n_sig_loc, 96), torch.uint8)
            if self.max_votes:
                s.v_sigs = self._zeros((self.n_sig_loc, 96), torch.uint8)
        self.h_members, self.h_off = np.asarray(members).astype(np.int64), off64

    def local_signatures(self, sigs):
        """The slice of an epoch's individual signatures (uint8[n_sig, 96], committee order) this rank aggregates."""
        return sigs[self.m0:self.m1]

    # ------------------------------------------------------------------ slashing detection
    def enable_slasher(self, history_epochs: int, max_attestations_per_target: int = None, current_epoch: int = 0, discount: bool = False):
        """Detect the double and surround votes of every accepted aggregate of every epoch processed from now on, against a history of
        `history_epochs` epochs on the device (Engine.slasher_init; B2Error(B2_ENOMEM) without allocating when it does not fit).
        Unsharded the history covers the whole registry; sharded, this rank's validators [v0, v1) only (6 * (v1 - v0) * H bytes).
        max_attestations_per_target defaults to 2 * n_agg, or 2 * max(n_agg, max_votes) with the vote form (at most 65535).  Every entry
        point then needs source_epoch (per aggregate) and current_epoch (the slasher's window moves to it before the epoch's update).
        The slasher is fed the epoch's signing roots as attestation roots, so it must not be shared with Spec.find_attester_slashings,
        which feeds data roots, on the same Engine.
        discount: every validator the slasher flags in an epoch becomes equivocating on the device right after that epoch's update
        (Engine.slasher_discount_dev, pos-evolution.md:1405-1461), so it counts in no head and moves no latest message from the next
        epoch on; Ticket.discounted() / discounted() name the newly marked validators, equivocating() reads the table."""
        n_val = self.n_val if self.n_val is not None else self.eng.n_validators
        v0, v1 = (self.v0, self.v1) if self.sharded else (0, n_val)
        K = min(2 * self.rows, 65535) if max_attestations_per_target is None else int(max_attestations_per_target)
        self.eng.slasher_init(n_val, history_epochs, K, current_epoch, v_begin=v0, v_end=v1)
        for s in self.slots:
            s.enable_slasher(self, discount)
        if discount and self.sharded and self.pg is not None:
            # this rank's slice of the equivocating table, padded to the longest range, and every rank's after the all-gather
            width = -(-n_val // self.world)
            self._eq_loc, self._eq_all = self._zeros(width, torch.uint8), self._zeros((self.world, width), torch.uint8)
        self.discount = bool(discount)
        self.sl_range = (v0, v1)
        self._sl_cur = self._sl_next = int(current_epoch)
        self.slasher = True

    def _slasher_args(self, source_epoch, current_epoch):
        """checked on entry, before anything of the epoch is enqueued"""
        if not self.slasher:
            return
        assert source_epoch is not None and current_epoch is not None, "the slasher is enabled: source_epoch and current_epoch are required"
        assert self._sl_next <= int(current_epoch) < 0xffffffff, "the slasher's current epoch only moves forward and fits 32 bits"
        self._sl_next = int(current_epoch)

    def _slasher_update(self, s, L, d_bits, d_msgs, d_source_epoch, d_target_epoch, current_epoch, host):
        """On the current stream, after the epoch's verdicts and fork choice: move the window if the epoch moved, then record and check
        ALL aggregates of the epoch with accept = the verdicts.  The roots are the epoch's signing roots, not the data roots the C ABI
        names: only attestations with the same target are compared for a double vote, and compute_signing_root(data,
        get_domain(DOMAIN_BEACON_ATTESTER, data.target.epoch)) uses one domain per target epoch on a chain, so two signing roots of one
        target are equal exactly when the data roots are (up to SHA-256 collisions)."""
        e = self.eng
        if int(current_epoch) != self._sl_cur:
            e.slasher_advance_dev(int(current_epoch))
            self._sl_cur = int(current_epoch)
        n = L.n
        e.slasher_update_dev(L.members, L.off, d_bits[:n], d_source_epoch[:n], d_target_epoch[:n], d_msgs[:n], s.ok[:n], s.sl_status[:n], s.sl_kind,
                             s.sl_conflict, s.sl_flagged)
        if host:
            s.h_sl_status[:n].copy_(s.sl_status[:n], non_blocking=True)
            s.h_sl_flagged.copy_(s.sl_flagged, non_blocking=True)

    def _discount(self, s, L, host):
        """On the current stream, after the epoch's slasher update: mark every flagged validator as equivocating.  Sharded, every rank
        marks its own range only; the ranks' range slices of the table are all-gathered and each other rank's range merged, so every
        replica holds the same table before the next epoch's exchange applies its latest messages."""
        e = self.eng
        e.slasher_discount_dev(L.members, s.sl_kind, s.sl_new, s.sl_n_new)
        if self.sharded and self.pg is not None:      # (bench.py --emulate-world: one rank on its own, nothing to gather)
            e.equivocating_slice_dev(self.v0, self.v1, self._eq_loc)
            torch.distributed.all_gather_into_tensor(self._eq_all.view(-1), self._eq_loc, group=self.pg)
            for g in range(self.world):
                if g != self.rank:
                    v0, v1 = g * self.n_val // self.world, (g + 1) * self.n_val // self.world
                    e.equivocating_merge_dev(v0, v1, self._eq_all[g])
        if host:
            s.h_sl_n_new.copy_(s.sl_n_new, non_blocking=True)

    def _read_discounted(self, s, host, event=None):
        if event is not None:
            event.synchronize()
        elif self.dev.type == "cuda":
            torch.cuda.current_stream().synchronize()
        n = int((s.h_sl_n_new if host else s.sl_n_new)[0])
        if n == 0:
            return np.zeros(0, dtype=np.int64)
        h_off, h_members, _ = self._host_layout(s)
        new = s.sl_new[:int(h_off[-1])].cpu().numpy()
        return np.sort(h_members[np.nonzero(new)[0]])

    def _host_layout(self, s):
        """(offsets, members, committee position of each member slot) of slot s's epoch on the host; in the vote form read back from the
        grouped arrays (the slot keeps them until it is claimed again)"""
        if not s.layout.votes:
            return self.h_off, self.h_members, None
        n = s.layout.n
        return (s.v_seg[:n + 1].cpu().numpy().astype(np.int64), s.v_members.cpu().numpy().astype(np.int64),
                s.v_pos.cpu().numpy().astype(np.int64))

    def discounted(self):
        """The validators the last epoch of process_epoch_dev / process_epoch_host newly marked as equivocating, sorted (synchronises the
        current stream)."""
        assert self.discount, "no discount: enable_slasher(..., discount=True)"
        return self._read_discounted(self.slots[0], False)

    def equivocating(self):
        """Store.equivocating_indices as uint8[n_validators] (nonzero = equivocating).  Needs a drained pipeline."""
        assert not self._inflight, "submitted epochs are in flight: drain() first"
        return self.eng.equivocating()

    def _read_slashings(self, s, host, event=None):
        """the findings in slot s as a Slashings tuple; kind and conflict targets cross to the host only when something was flagged"""
        if event is not None:
            event.synchronize()
        elif self.dev.type == "cuda":
            torch.cuda.current_stream().synchronize()
        rows = s.layout.n
        if host:
            status, n = s.h_sl_status[:rows].numpy().copy(), int(s.h_sl_flagged[0])
        else:
            status, n = s.sl_status[:rows].cpu().numpy(), int(s.sl_flagged[0])
        if n == 0:
            none = np.zeros(0, dtype=np.int64)
            return Slashings(status, none, none, none, np.zeros(0, np.uint8), np.zeros(0, np.uint32), np.zeros(0, np.uint32))
        h_off, h_members, h_pos = self._host_layout(s)
        total = int(h_off[-1])
        kind = s.sl_kind[:total].cpu().numpy()
        conflict = s.sl_conflict[:total].cpu().numpy().view(np.uint32)
        i = np.nonzero(kind)[0]
        agg = np.searchsorted(h_off, i, side="right") - 1
        # vote form: `aggregate` is the vote id and `position` the member's position in its committee
        pos = i - h_off[agg] if h_pos is None else h_pos[i]
        return Slashings(status, agg, pos, h_members[i], kind[i], conflict[i, 0].copy(), conflict[i, 1].copy())

    def slashings(self) -> Slashings:
        """The slasher's findings for the last epoch of process_epoch_dev / process_epoch_host (synchronises the current stream)."""
        assert self.slasher, "no slasher: enable_slasher"
        return self._read_slashings(self.slots[0], False)

    # ------------------------------------------------------------------ the exchange + fork choice of one epoch
    def _exchange(self, s, L, d_bits, d_target_epoch, d_block_idx):
        """Sharded epoch, after the local tail: all-gather (aggregate signature, verdict) of every rank's aggregates, then
        update_latest_messages for ALL accepted aggregates of the epoch on this rank's replica of the LMD table."""
        p = L.pad
        if self.pg is None:                           # one rank of a sharded epoch on its own (bench.py --emulate-world): no peers to gather from
            L.out_all[self.rank].copy_(L.out_loc)
        else:
            torch.distributed.all_gather_into_tensor(L.out_all.view(-1), L.out_loc, group=self.pg)
        if L.ranges is None:                          # committee form: every rank holds n_loc aggregates
            s.agg_sig[:L.n].view(self.world, p * 96).copy_(L.out_all[:, :p * 96])
            s.ok[:L.n].view(self.world, p).copy_(L.out_all[:, p * 96:])
        else:                                         # vote form: rank g's count of votes, from its first vote on
            for g, (r0, k) in enumerate(L.ranges):
                s.agg_sig[r0:r0 + k].view(-1).copy_(L.out_all[g, :k * 96])
                s.ok[r0:r0 + k].copy_(L.out_all[g, p * 96:p * 96 + k])
        n = L.n
        self.eng.latest_messages_update_dev(L.members, L.off, d_bits[:n], d_target_epoch[:n], d_block_idx[:n], s.ok[:n])

    def _fork_choice(self, s, justified_idx, boost_idx, boost_score):
        e = self.eng
        if self.sharded:
            e.vote_weights_range_dev(self.v0, self.v1, self.d_votes)
        else:
            e.vote_weights_dev(self.d_votes)
        if self.pg is not None and torch.distributed.get_world_size(self.pg) > 1:
            torch.distributed.all_reduce(self.d_votes, group=self.pg)
        e.head_from_votes_dev(self.d_votes, s.head, justified_idx, boost_idx, boost_score)

    def enable_fused_get_head(self):
        """Sharded mode: set up get_head as ONE kernel per rank with the vote all-reduce fused in over NVLink peer memory
        (Engine.fc_exchange_setup: CUDA IPC handles exchanged over the process group).  Call on every rank, after tree_load."""
        assert self.sharded, "the fused multi-GPU get_head is for a validator set sharded over the ranks"
        ok, why = 1, ""
        try:
            self.eng.fc_exchange_setup(self.rank, self.world, self.pg)
        except Exception as e:                        # e.g. CUDA IPC not permitted between the processes of this box
            ok, why = 0, repr(e)
        flag = torch.tensor([ok], dtype=torch.int32, device=self.dev)
        torch.distributed.all_reduce(flag, op=torch.distributed.ReduceOp.MIN, group=self.pg)      # all ranks or none: the call is collective
        self._fused_head = bool(int(flag.item()))
        self.fused_head_error = why
        return self._fused_head

    # ------------------------------------------------------------------ changing the block tree between batches
    def _check_tree(self):
        """The vote scatter writes one entry per block of the engine's tree into d_votes: refuse before anything is enqueued when the
        tree's size is not the one d_votes was sized for (a tree_load behind the processor's back; add_blocks / prune_tree re-size it)."""
        if isinstance(self.eng, Engine) and self.eng.tree_size() != self.d_votes.numel():
            raise ValueError("the engine's tree has %d blocks but this EpochProcessor's vote vector %d: change the tree through "
                             "add_blocks / prune_tree" % (self.eng.tree_size(), self.d_votes.numel()))

    def _tree_changed(self):
        n = self.eng.tree_size()
        if n != self.d_votes.numel():
            self.d_votes = self._zeros(n, torch.int64)
            self.n_blocks = n
            self._fused_head = False          # the NVLink exchange block is sized by the tree: enable_fused_get_head again
        return n

    def add_blocks(self, parent, slot, roots32, leaf_viable):
        """Engine.tree_add between batches (on_block); needs a drained pipeline."""
        assert not self._inflight, "submitted epochs are in flight: drain() first"
        self.eng.tree_add(parent, slot, roots32, leaf_viable)
        self._tree_changed()

    def prune_tree(self, new_root):
        """Engine.tree_prune between batches (finalization): returns the map old id -> new id; block indices of later epochs use the new
        ids.  Needs a drained pipeline."""
        assert not self._inflight, "submitted epochs are in flight: drain() first"
        m = self.eng.tree_prune(new_root)
        self._tree_changed()
        return m

    def set_viable(self, idx, viable):
        """Engine.tree_set_viable between batches; needs a drained pipeline."""
        assert not self._inflight, "submitted epochs are in flight: drain() first"
        self.eng.tree_set_viable(idx, viable)

    def get_head(self, justified_idx=0, boost_idx=-1, boost_score=0, fused=None):
        """get_head over the current LMD table through the multi-rank path; returns the head index on the host.  COLLECTIVE.
        fused (default: whether enable_fused_get_head was called): one kernel per rank -- vote scatter of this rank's validators,
        64-bit reductions into every rank's accumulator over NVLink, flag exchange, tree phase, zero-copy result.  Otherwise the
        three-stage form: scatter kernel, NCCL all-reduce of u64[n_blocks], tree kernel, device-to-host copy.  Needs a drained pipeline."""
        assert not self._inflight, "submitted epochs are in flight: drain() first"
        self._check_tree()
        if fused is None:
            fused = getattr(self, "_fused_head", False)
        if fused:
            return self.eng.get_head_multi(self.v0, self.v1, justified_idx, boost_idx, boost_score)
        self._fork_choice(self.slots[0], justified_idx, boost_idx, boost_score)
        return int(self.slots[0].head.item())

    # ------------------------------------------------------------------ one epoch, both forms
    def _stage(self, s, host, sigs, bits, msgs, tgt, blk, src, n=None):
        """Copy an epoch's inputs into slot s on the current stream; returns (sigs, bits, msgs, tgt, blk, src) with each copied array
        replaced by the slot's.  From the host everything is copied.  From the device only what the asynchronous tail reads after
        the call has returned: the target epochs and block indices of the LMD update (a caller may rewrite them for the next epoch),
        and with the slasher the bits, messages and source epochs, which its update reads after the ticket's event.  n: rows (default
        n_agg).  The vote form passes bits=None: the grouping writes the slot's bit rows."""
        n = self.n_agg if n is None else n

        def put(buf, a):
            if a is None:
                return buf[:n]
            buf[:n].copy_(a, non_blocking=True)
            return buf[:n]
        if host:
            sigs, bits, msgs = s.sigs.copy_(sigs, non_blocking=True), put(s.bits, bits), put(s.msgs, msgs)
        tgt, blk = put(s.tgt, tgt), put(s.blk, blk)
        if self.slasher:
            if not host:
                bits, msgs = put(s.bits, bits), put(s.msgs, msgs)
            src = put(s.src, src)
        return sigs, bits, msgs, tgt, blk, src

    # ------------------------------------------------------------------ vote form
    def _votes_check(self, votes):
        """Host checks of votes=(vote, vote_off), before anything of the epoch is enqueued; returns (vote, vote_off as int64, n_votes)."""
        if self.max_votes is None:
            raise ValueError("votes= needs an EpochProcessor constructed with max_votes")
        vote, vote_off = votes
        vo = np.asarray(vote_off).astype(np.int64)
        if vo.shape != (self.n_agg + 1,) or vo[0] != 0 or np.any(np.diff(vo) <= 0):
            raise ValueError("vote_off must hold n_committees + 1 = %d entries, start at 0 and increase strictly" % (self.n_agg + 1))
        if np.any(np.diff(vo) > 8 * self.bits_stride):
            raise ValueError("a committee has more vote ids than its bit row has positions (8 * bits_stride)")
        n_votes = int(vo[-1])
        if n_votes > self.max_votes:
            raise ValueError("the epoch has %d votes, more than max_votes = %d" % (n_votes, self.max_votes))
        if tuple(vote.shape) != (self.n_sig,) or vote.element_size() != 4:
            raise ValueError("vote must hold one 32-bit id per member of the epoch (%d)" % self.n_sig)
        return vote, vo, n_votes

    def _committee_layout(self, s, sigs):
        sh = self.sharded
        return _Layout(False, self.n_agg, self.d_members, self.d_off, self.a0, self.a1, self.d_members_loc if sh else None, self.d_off_loc if sh else None,
                       sigs, self.n_loc, None, s.out_loc if sh else None, s.out_all if sh else None)

    def _group(self, s, vote, vo, n_votes, sigs):
        """On the current stream (the one that claimed slot s): upload vote_off, group the epoch by vote into the slot's buffers, and
        return the epoch's _Layout over them."""
        e = self.eng
        if s.ev_vote_off is not None:
            s.ev_vote_off.synchronize()               # the slot's previous upload has left the pinned buffer
        s.h_vote_off.copy_(torch.from_numpy(vo.astype(np.int32)))
        s.v_vote_off.copy_(s.h_vote_off, non_blocking=True)
        if self.dev.type == "cuda":
            s.ev_vote_off = self._record()
        seg = s.v_seg[:n_votes + 1]
        e.votes_group_dev(vote, s.v_vote_off, self.d_members, self.d_off, sigs, self.a0, self.a1, s.v_sigs, s.v_members, s.v_pos, seg,
                          s.bits[:n_votes], s.v_aggbits[:n_votes], d_seg_off_loc=s.v_seg_loc if self.sharded else None)
        r0, r1 = int(vo[self.a0]), int(vo[self.a1])
        if not self.sharded:
            return _Layout(True, n_votes, s.v_members, seg, r0, r1, None, None, s.v_sigs, None, None, None, None)
        ranges = [(int(vo[g * self.n_agg // self.world]), int(vo[(g + 1) * self.n_agg // self.world] - vo[g * self.n_agg // self.world]))
                  for g in range(self.world)]
        p = max(k for _, k in ranges)
        return _Layout(True, n_votes, s.v_members, seg, r0, r1, s.v_members[self.m0:self.m1], s.v_seg_loc[:r1 - r0 + 1], s.v_sigs, p, ranges,
                       s.vout_loc[:p * 97], s.vout_all[:self.world * p * 97].view(self.world, p * 97))

    @staticmethod
    def _record():
        ev = torch.cuda.Event()
        ev.record()
        return ev

    def _epoch(self, s, L, x, fc, host, current_epoch, pipelined, last=False):
        """The epoch of slot s with inputs x = (sigs, bits, msgs, tgt, blk, src): verify, exchange (sharded), fork choice (fc =
        justified_idx, boost_idx, boost_score), host readback (host), slasher update.  Synchronous: Engine.epoch_dev and the rest on the
        current stream.  Pipelined: epoch_start_dev / epoch_tail_dev on the current stream, then the rest on the fork-choice stream
        after epoch_wait_dev, enqueued BEFORE the next epoch's tail (whose LMD update waits for this scatter), recording the slot's
        events."""
        e = self.eng
        s.layout = L
        sigs, bits, msgs, tgt, blk, src = x
        if self.sharded:                                  # this rank's aggregates; their LMD update waits for the exchange
            n = L.r1 - L.r0
            members, off, v_bits, v_msgs, v_tgt, v_blk = L.members_loc, L.off_loc, bits[L.r0:L.r1], msgs[L.r0:L.r1], None, None
            o_sig, o_ok = L.out_loc[:n * 96], L.out_loc[L.pad * 96:L.pad * 96 + n]
        else:
            n = L.n
            members, off, v_bits, v_msgs, v_tgt, v_blk = L.members, L.off, bits[:n], msgs[:n], tgt[:n], blk[:n]
            o_sig, o_ok = s.agg_sig[:n], s.ok[:n]
        sigs = L.sigs
        if pipelined:
            team = last or self.always_team
            if team != self._team_form:                   # last epoch of a batch: nothing will overlap its tail, so take the short form
                e.epoch_set_pairing_form(team)
                self._team_form = team
            e.epoch_start_dev(s.i, sigs, members, off, v_bits, v_msgs, s.agg_status)
            e.epoch_tail_dev(s.i, members, off, v_bits, v_tgt, v_blk, o_sig, s.agg_status, o_ok)
        else:
            e.epoch_dev(sigs, members, off, v_bits, v_msgs, v_tgt, v_blk, o_sig, s.agg_status, o_ok)
        with torch.cuda.stream(self.fc_stream) if pipelined else contextlib.nullcontext():
            if pipelined:
                e.epoch_wait_dev(s.i)
            if L.votes:                                   # this rank's votes without attester read as empty segments
                e.votes_empty_dev(v_bits, o_sig, s.agg_status[:n])
            if self.sharded:
                self._exchange(s, L, bits, tgt, blk)
            self._fork_choice(s, *fc)
            if host:
                s.h_ok[:L.n].copy_(s.ok[:L.n], non_blocking=True)
                s.h_head.copy_(s.head, non_blocking=True)
                s.h_agg_sig[:L.n].copy_(s.agg_sig[:L.n], non_blocking=True)
                if L.votes:
                    s.h_aggbits[:L.n].copy_(s.v_aggbits[:L.n], non_blocking=True)
            if pipelined:
                s.ev_fc = self._record()
            if self.slasher:                              # after the head: the head's latency does not include it
                self._slasher_update(s, L, bits, msgs, src, tgt, current_epoch, host)
                if self.discount:                         # before the next epoch's LMD update and head (the library orders its tail)
                    self._discount(s, L, host)
                if pipelined:
                    s.ev_sl = self._record()

    # ------------------------------------------------------------------ attestation intake
    def intake_dev(self, d_wire, d_woff, epoch, current_slot, domain32, committees_per_slot, slots_per_epoch) -> Intake:
        """One epoch of unaggregated Attestations straight off the wire (d_wire uint8, d_woff int32/uint32[n_att + 1] on the device, the
        form of Engine.attestations_decode) checked against the device tree and turned into the vote form's inputs for this processor's
        committees (Engine.attestation_intake_dev, on the current stream).  Returns an Intake of fresh tensors, which follow the input
        contract of submit_dev once submitted.  Reading vote_off waits for the current stream's work up to the intake: enqueue it under a
        stream that carries no epoch (torch.cuda.stream(...)) and it waits for the intake alone.  An epoch with more than max_votes votes
        is then refused by submit_dev.  Not for a sharded processor."""
        def call(r, d_vote_off):
            self.eng.attestation_intake_dev(d_wire, d_woff, self.d_off, epoch, current_slot, domain32, committees_per_slot, slots_per_epoch,
                                            self.bits_stride, r.status, r.vote, d_vote_off, r.sigs, r.data128, r.msgs, r.source_epoch,
                                            r.target_epoch, r.block_idx)
        return self._intake("intake_dev", call, d_woff.numel() - 1, committees_per_slot, slots_per_epoch)

    def intake_single_dev(self, d_wire, d_woff, d_subnet, epoch, current_slot, domain32, committees_per_slot, slots_per_epoch,
                          subnet_count=64) -> Intake:
        """intake_dev for one epoch of Electra SingleAttestations (240-byte encodings on the device, d_woff their offsets, d_subnet
        int32/uint32[n_att] the subnet each arrived on, subnet_count = ATTESTATION_SUBNET_COUNT) against this processor's committees
        (Engine.single_attestation_intake_dev, on the current stream).  The same Intake, contract and refusals as intake_dev; status holds
        b2_single_attestation_intake's statuses."""
        def call(r, d_vote_off):
            self.eng.single_attestation_intake_dev(d_wire, d_woff, d_subnet, self.d_members, self.d_off, epoch, current_slot, domain32,
                                                   committees_per_slot, slots_per_epoch, self.bits_stride, r.status, r.vote, d_vote_off, r.sigs,
                                                   r.data128, r.msgs, r.source_epoch, r.target_epoch, r.block_idx, subnet_count=subnet_count)
        return self._intake("intake_single_dev", call, d_woff.numel() - 1, committees_per_slot, slots_per_epoch)

    def _intake(self, name, call, n_att, committees_per_slot, slots_per_epoch) -> Intake:
        """Both intakes: the refusals, fresh outputs, call(outputs, d_vote_off) on the current stream, then vote_off on the host"""
        if self.sharded:
            raise ValueError("%s: a sharded EpochProcessor is not supported" % name)
        if self.max_votes is None:
            raise ValueError("%s needs an EpochProcessor constructed with max_votes" % name)
        if int(committees_per_slot) * int(slots_per_epoch) != self.n_agg:
            raise ValueError("committees_per_slot * slots_per_epoch must be the processor's n_agg = %d" % self.n_agg)
        self._check_tree()
        z, mv = self._zeros, self.max_votes
        r = Intake(z((self.n_sig, 96), torch.uint8), torch.full((self.n_sig,), -1, dtype=torch.int32, device=self.dev), z((mv, 32), torch.uint8),
                   z(mv, torch.int64), z(mv, torch.int32), z(mv, torch.int64), z((mv, 128), torch.uint8), z(n_att, torch.int32), None)
        d_vote_off = z(self.n_agg + 1, torch.int32)
        call(r, d_vote_off)
        h = self._pinned(self.n_agg + 1, torch.int32)
        h.copy_(d_vote_off, non_blocking=True)
        self._record().synchronize()
        vote_off = h.numpy().astype(np.int64)
        n = min(int(vote_off[-1]), mv)                  # the per-vote rows the entry points take: one per vote
        return r._replace(msgs=r.msgs[:n], target_epoch=r.target_epoch[:n], block_idx=r.block_idx[:n], source_epoch=r.source_epoch[:n],
                          data128=r.data128[:n], vote_off=vote_off)

    # ------------------------------------------------------------------ synchronous form
    def _prepare(self, s, host, sigs, bits, msgs, tgt, blk, src, V):
        """Stage slot s's inputs on the current stream and, in the vote form (V = _votes_check's result), group the epoch there; returns
        (layout, staged inputs)."""
        if V is None:
            x = self._stage(s, host, sigs, bits, msgs, tgt, blk, src)
            return self._committee_layout(s, x[0]), x
        vote, vo, n_votes = V
        x = self._stage(s, host, sigs, None, msgs, tgt, blk, src, n=n_votes)
        x = (x[0], s.bits[:n_votes]) + x[2:]            # the grouping writes the bit rows
        if host:
            vote = s.v_vote.copy_(vote, non_blocking=True)
        return self._group(s, vote, vo, n_votes, x[0]), x

    def process_epoch_dev(self, d_sigs, d_bits, d_msgs, d_target_epoch, d_block_idx, justified_idx=0, boost_idx=-1, boost_score=0,
                          source_epoch=None, current_epoch=None, votes=None):
        """d_sigs: this rank's signatures (all of them when not sharded); every other array covers the whole epoch.  With the slasher
        on: source_epoch int64[n_agg] (device) and the current epoch; the findings are read with slashings().  Needs a drained pipeline.
        votes=(vote, vote_off): the vote form (module docstring): vote int32/uint32[n_sig] on the device, vote_off on the host; d_bits is
        then unused (None) and d_msgs, d_target_epoch, d_block_idx and source_epoch hold one row per vote."""
        assert not self._inflight, "submitted epochs are in flight: drain() first"
        self._check_tree()
        self._slasher_args(source_epoch, current_epoch)
        V = None if votes is None else self._votes_check(votes)
        s = self.slots[0]
        L, x = self._prepare(s, False, d_sigs, d_bits, d_msgs, d_target_epoch, d_block_idx, source_epoch, V)
        self._epoch(s, L, x, (justified_idx, boost_idx, boost_score), False, current_epoch, pipelined=False)
        return s.ok[:L.n], s.head

    def process_epoch_host(self, h_sigs, h_bits, h_msgs, h_target_epoch, h_block_idx, justified_idx=0, boost_idx=-1, boost_score=0,
                           source_epoch=None, current_epoch=None, votes=None):
        """Pinned host tensors in, (verdict bytes, head index) out on the host; returns when the epoch is done.  With the slasher on:
        source_epoch int64[n_agg] (pinned host) and the current epoch; the findings are read with slashings().  Needs a drained
        pipeline.  votes=(vote, vote_off): the vote form, vote as a pinned host tensor (see process_epoch_dev)."""
        assert not self._inflight, "submitted epochs are in flight: drain() first"
        self._check_tree()
        self._slasher_args(source_epoch, current_epoch)
        V = None if votes is None else self._votes_check(votes)
        s = self.slots[0]
        L, x = self._prepare(s, True, h_sigs, h_bits, h_msgs, h_target_epoch, h_block_idx, source_epoch, V)
        self._epoch(s, L, x, (justified_idx, boost_idx, boost_score), True, current_epoch, pipelined=False)
        torch.cuda.current_stream().synchronize()
        return s.h_ok[:L.n], int(s.h_head[0])

    # ------------------------------------------------------------------ pipelined form
    def _submit(self, s, L, x, fc, host, last, current_epoch):
        self._epoch(s, L, x, fc, host, current_epoch, pipelined=True, last=last)
        self._inflight.append(_Ticket(self, s, host))
        self.k += 1
        return self._inflight.popleft() if len(self._inflight) >= self.depth else None

    def _claim_slot(self, stream):
        """`stream` is about to overwrite the slot's inputs/outputs: its previous epoch (tail and fork choice) must be done."""
        s = self.slots[self.k % self.depth]
        self.eng.epoch_wait_dev(s.i)                      # (on the current stream == `stream`)
        if s.ev_fc is not None:
            stream.wait_event(s.ev_fc)
        if s.ev_sl is not None:                           # the slasher read the slot's bits, messages, epochs and verdicts
            stream.wait_event(s.ev_sl)
        return s

    def drain_hint(self, remaining: int) -> bool:
        """True when an epoch with `remaining` epochs still to come after it should take the short-latency (team) tail: the last epochs
        of a batch cannot hide a thread-form tail (≈ 30 ms) behind decompressions that are no longer coming."""
        return remaining < self.team_last

    def submit_dev(self, d_sigs, d_bits, d_msgs, d_target_epoch, d_block_idx, justified_idx=0, boost_idx=-1, boost_score=0, last=False,
                   source_epoch=None, current_epoch=None, votes=None):
        """Enqueue one epoch (device-resident inputs, which must stay untouched until its ticket has been waited for; d_sigs =
        this rank's signatures, the other arrays cover the whole epoch).  Returns the ticket of the epoch submitted depth-1
        calls earlier (None while the pipeline fills).  `last=True` says no further epoch follows soon: its pairing tail is
        enqueued in the short-critical-path (team) form.  With the slasher on: source_epoch int64[n_agg] (device) and the
        current epoch; the slasher reads copies of the bits, messages and epochs, so the inputs are free after wait() as without it.
        votes=(vote, vote_off): the vote form (see process_epoch_dev); the grouping runs on the current stream after the slot is claimed."""
        self._check_tree()
        self._slasher_args(source_epoch, current_epoch)
        V = None if votes is None else self._votes_check(votes)
        s = self._claim_slot(torch.cuda.current_stream())
        L, x = self._prepare(s, False, d_sigs, d_bits, d_msgs, d_target_epoch, d_block_idx, source_epoch, V)
        return self._submit(s, L, x, (justified_idx, boost_idx, boost_score), False, last, current_epoch)

    def submit_host(self, h_sigs, h_bits, h_msgs, h_target_epoch, h_block_idx, justified_idx=0, boost_idx=-1, boost_score=0, last=False,
                    source_epoch=None, current_epoch=None, votes=None):
        """Pinned host tensors in (untouched until the returned-later ticket has been waited for).  The H2D copies go on a
        separate stream so that they overlap with the epochs in flight.  With the slasher on: source_epoch int64[n_agg] (pinned
        host) and the current epoch; the status and flagged count of every epoch come back in pinned buffers.  votes=(vote, vote_off):
        the vote form, vote as a pinned host tensor; it is grouped on the copy stream after the H2D copies."""
        self._check_tree()
        self._slasher_args(source_epoch, current_epoch)
        V = None if votes is None else self._votes_check(votes)
        cur = torch.cuda.current_stream()
        with torch.cuda.stream(self.copy_stream):
            s = self._claim_slot(self.copy_stream)
            L, x = self._prepare(s, True, h_sigs, h_bits, h_msgs, h_target_epoch, h_block_idx, source_epoch, V)
            ev = self._record()
        cur.wait_event(ev)
        return self._submit(s, L, x, (justified_idx, boost_idx, boost_score), True, last, current_epoch)

    def drain(self):
        """Tickets of the epochs still in flight, oldest first; the current stream waits for all of them (their slasher updates included)."""
        out = list(self._inflight)
        self._inflight.clear()
        for t in out:
            torch.cuda.current_stream().wait_event(t.event)
            if t.slasher_event is not None:
                torch.cuda.current_stream().wait_event(t.slasher_event)
        return out

    @property
    def h2d_bytes(self):
        """host -> device bytes per epoch of this rank (submit_host): its signatures + the epoch's bits, messages, epochs, blocks"""
        n = self.n_agg
        return self.slots[0].sigs.numel() + n * (self.bits_stride + 32 + 8 + 4) + (8 * n if self.slasher else 0)

    @property
    def d2h_bytes(self):
        """device -> host bytes per epoch (submit_host): verdicts + head index + the aggregate signatures (+ the slasher's statuses and
        flagged count, and with the discount its newly-marked count; its kind and conflict targets only when something was flagged)"""
        return self.n_agg * 97 + 4 + ((4 * self.n_agg + 4) if self.slasher else 0) + (4 if self.discount else 0)
