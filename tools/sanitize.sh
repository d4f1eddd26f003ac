#!/bin/bash
# tools/sanitize.sh -- SURVEY.md section 5 tooling, run on a GPU machine (bash tools/sanitize.sh); logs -> $OUT (default: a temporary directory) (copy
# the summaries wherever they are kept).
#   1. compute-sanitizer --tool memcheck   over the small-configuration GPU tests (every kernel, out-of-bounds / misaligned accesses)
#   2. compute-sanitizer --tool racecheck  over the tests whose kernels share data through shared memory: the 3-lane team pairing
#      (__syncwarp between phases), the TMA-staged gather (mbarrier + cp.async.bulk), the vote scatter's shared bins, the tree kernel,
#      the block packer's per-committee fold and greedy, the SSZ leaf staging and subtree reduction, the intake's per-committee grouping
#      (ldata, win, first) on colliding data
#   3. compute-sanitizer --tool synccheck  on the same subset (illegal barrier use)
#   4. the host side of the C ABI under AddressSanitizer + UBSan (pos_evolution_b200/libb200pos_asan.so, built by
#      `python -m pos_evolution_b200.build --asan`) over the BLS / fork-choice / guard / error-contract tests and the argument checks both
#      forms of each entry point share
set -u
cd "$(dirname "$0")/.."
OUT="${OUT:-$(mktemp -d)}"
mkdir -p "$OUT"
SAN=/usr/local/cuda/bin/compute-sanitizer
SMALL="tests/test_gpu_bls.py tests/test_gpu_bls_adversarial.py tests/test_gpu_aggregate_verify.py tests/test_gpu_sync_aggregate.py tests/test_gpu_forkchoice.py tests/test_gpu_gather.py tests/test_gpu_participation.py tests/test_gpu_epoch.py tests/test_gpu_slasher.py tests/test_gpu_epoch_slasher.py tests/test_gpu_epoch_votes.py tests/test_gpu_intake.py::test_every_status_and_output_matches_oracle tests/test_gpu_intake.py::test_device_guards tests/test_gpu_intake.py::test_rejected_host_calls_change_nothing tests/test_gpu_intake_shapes.py::test_single_committee_epoch tests/test_gpu_intake_shapes.py::test_more_than_1024_committees tests/test_gpu_intake_shapes.py::test_votes_group_matches_numpy_model tests/test_gpu_epoch_discount.py tests/test_gpu_pack.py tests/test_gpu_ssz.py::test_validators_load tests/test_gpu_ssz.py::test_incremental_updates tests/test_gpu_tree_update.py::test_random_sequences_match_a_fresh_load tests/test_gpu_tree_update.py::test_root_ties tests/test_gpu_tree_update.py::test_rejected_calls_change_nothing tests/test_gpu_intake_keys.py::test_intake_collision_sets[64-33] tests/test_gpu_intake_keys.py::test_intake_collision_sets[2048-2] tests/test_gpu_intake_keys.py::test_aggregate_data_table[3-False] tests/test_gpu_intake_keys.py::test_aggregate_data_table[65-False] tests/test_gpu_intake_keys.py::test_roots[one_block] tests/test_gpu_intake_keys.py::test_colliding_votes_end_to_end"
RACE="tests/test_gpu_bls.py::test_fast_aggregate_verify_vs_oracle tests/test_gpu_bls.py::test_g1_aggregate_all_minimal_committees tests/test_gpu_forkchoice.py tests/test_gpu_gather.py tests/test_gpu_pack.py::test_pack_matches_oracle tests/test_gpu_ssz.py::test_validators_load tests/test_gpu_intake_keys.py::test_intake_collision_sets[64-33] tests/test_gpu_intake_keys.py::test_intake_collision_sets[2048-2]"
run() {  # name, timeout, command...
    local name=$1 tmo=$2; shift 2
    echo "== $name"
    timeout "$tmo" "$@" > "$OUT/sanitize_$name.log" 2>&1
    echo "rc=$? ($name)"; grep -E "ERROR SUMMARY|RACECHECK SUMMARY|passed|failed|error" "$OUT/sanitize_$name.log" | tail -6
}
run memcheck 600 $SAN --tool memcheck --error-exitcode 1 --launch-timeout 600 python -m pytest $SMALL -x -q -m gpu -k "not test_epoch_pipeline or sync-3 or pipelined-3 or pipelined_rlc or pipelined_team"
run racecheck 420 $SAN --tool racecheck --racecheck-report all --error-exitcode 1 python -m pytest $RACE -x -q -m gpu
run synccheck 300 $SAN --tool synccheck --error-exitcode 1 python -m pytest $RACE -x -q -m gpu
if [ -f pos_evolution_b200/libb200pos_asan.so ]; then
    ASAN_LIB=$(gcc -print-file-name=libasan.so)
    B2_LIB=$PWD/pos_evolution_b200/libb200pos_asan.so LD_PRELOAD=$ASAN_LIB ASAN_OPTIONS=protect_shadow_gap=0:detect_leaks=0:halt_on_error=1 UBSAN_OPTIONS=print_stacktrace=1 \
        run asan_host 300 python -m pytest tests/test_gpu_bls.py tests/test_gpu_forkchoice.py tests/test_gpu_gather.py tests/test_gpu_participation.py \
        tests/test_gpu_abi_contract.py tests/test_gpu_abi_pairs.py -x -q -m gpu
else
    echo "no ASan build (python -m pos_evolution_b200.build --asan)"
fi
