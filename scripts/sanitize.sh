#!/bin/bash
# compute-sanitizer over one run of every kernel family (SURVEY section 5 / VERDICT r1 item 10).  Logs -> gpurun_out/.
#   bash scripts/sanitize.sh            (on the GPU box, from the repo root)
OUT=${1:-gpurun_out}
mkdir -p "$OUT"
SAN=/usr/local/cuda/bin/compute-sanitizer
SEL_HMC="tests/test_hmc_gpu.py tests/test_sink_gpu.py"
SEL_RM="tests/test_rmhmc_gpu.py -k funnel2-or-funnel32-or-full48-or-jacdiag-or-standalone"
run() {   # tool, tag, timeout, pytest args...
    local tool=$1 tag=$2 to=$3; shift 3
    timeout "$to" $SAN --tool "$tool" --print-limit 20 --error-exitcode 0 --log-file "$OUT/san_${tool}_${tag}.log" \
        python -m pytest "$@" -x -q -p no:cacheprovider > "$OUT/san_${tool}_${tag}.pytest.log" 2>&1
    echo "$tool $tag: rc=$? $(tail -1 "$OUT/san_${tool}_${tag}.pytest.log") | $(grep -E 'ERROR SUMMARY|RACECHECK SUMMARY' "$OUT/san_${tool}_${tag}.log" | tail -1)"
}
if [ -z "${SAN_ONLY:-}" ]; then
run memcheck hmc 500 tests/test_hmc_gpu.py tests/test_sink_gpu.py
run memcheck rmhmc 500 tests/test_rmhmc_gpu.py -k "funnel2 or funnel32 or full48 or jacdiag or standalone"
run memcheck mlp 500 tests/test_mlp_gpu.py tests/test_mlp_tc_gpu.py -k "split_sym or mlp_full or chain_parity"
run memcheck dense 500 tests/test_tc_gpu.py tests/test_rmhmc_dense_gpu.py -k "edge_shapes or parity"
run racecheck hmc 400 tests/test_hmc_gpu.py -k "iso256 or nuts or reversib"
run racecheck rmhmc 400 tests/test_rmhmc_gpu.py -k "funnel2 or funnel32"
run racecheck mlp 400 tests/test_mlp_tc_gpu.py -k "chain_parity"
run racecheck dense 400 tests/test_tc_gpu.py -k "edge_shapes"
run memcheck rank 500 tests/test_rank_diagnostics_gpu.py -k "edge_case or duplicates or slab or odd_dimension"
run racecheck rank 400 tests/test_rank_diagnostics_gpu.py -k "edge_case or duplicates"
run synccheck all 400 tests/test_hmc_gpu.py tests/test_rmhmc_gpu.py tests/test_mlp_tc_gpu.py -k "iso256 or funnel2 or funnel32 or chain_parity"
fi
# the persistent small-D flow kernel (hmcx_flow.cu): golden chains, live-oracle RMHMC, ragged shapes, all chains-per-warp forms
if [ "${SAN_ONLY:-}" = "flow" ] || [ -z "${SAN_ONLY:-}" ]; then
run memcheck flow 500 tests/test_rmhmc_dense_gpu.py tests/test_tc_gpu.py tests/test_hmc_gpu.py -k "flow or (golden_chain_parity and (full48 or full40 or iso40 or blockmass) and not tcgen05) or paths_agree"
run racecheck flow 500 tests/test_rmhmc_dense_gpu.py tests/test_tc_gpu.py -k "(flow and not statistics) or paths_agree"
fi
# later in round 2: windowed delivery (two streams + hmcx_copy_rows_async) and the split schedule's gradient re-use (cluster
# barrier arrive / wait pairing at the positions that skip their evaluation or their kick)
if [ "${SAN_ONLY:-}" = "late" ] || [ -z "${SAN_ONLY:-}" ]; then
run memcheck windows 300 tests/test_sink_gpu.py -k "windowed"
run synccheck reuse 500 tests/test_mlp_gpu.py -k "cluster_split or split_sym or split_kmid"
run memcheck reuse 500 tests/test_mlp_gpu.py -k "cluster_split or split_sym or split_kmid"
fi
