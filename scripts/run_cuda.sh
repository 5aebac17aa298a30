#!/usr/bin/env bash
# Sweep the concurrency benchmark (CUDA backend) over an environment matrix x modes x the
# five command groups, log everything, print the SUCCESS/FAILURE tables.
# Role of concurency/run_sycl.sh in the reference; the Level-Zero / SYCL plugin knobs become
# their CUDA analogues (HW-queue count, copy engine vs SM copy in the fused kernel, device choice).
set -o xtrace
here="$(cd "$(dirname "${BASH_SOURCE[0]}")/.." && pwd)"
make -C "$here" -j bin/concurency >/dev/null || exit 1
work=$(mktemp -d tmp-cuda-XXXX); cd "$work" || exit 1
rm -f cuda.log

LCOMMANDS=("C C" "C M2D" "C D2M" "M2D D2M" "H2D D2H")
EXTRA=("C D2P" "D2P P2D" "A H2D")          # beyond the reference: peer-GPU copies, stream-triad compute
MODES=(${HPCP_CUDA_MODES:-out_of_order in_order host_threads nowait fused})
# HPCP_CUDA_ELEMS shrinks the copies (default: the reference's 1 GB); without a GPU the binary falls back to
# its CPU backend, which only has host_threads / nowait (HPCP_CUDA_MODES="host_threads nowait").
SIZE_ARGS=(${HPCP_CUDA_ELEMS:+--globalsize_default_memory $HPCP_CUDA_ELEMS})

for envs in "HPCP_DEVICE=0" \
            "HPCP_DEVICE=0 CUDA_DEVICE_MAX_CONNECTIONS=1" \
            "HPCP_DEVICE=0 CUDA_DEVICE_MAX_CONNECTIONS=32" \
            "HPCP_DEVICE=0 HPCP_FUSED_COPY_ENGINE=ldst"
do
    (
    export $envs
    for mode in "${MODES[@]}"; do
        # shellcheck disable=SC2068,SC2086
        "$here/bin/concurency" "$mode" ${LCOMMANDS[@]/#/--commands } ${EXTRA_GROUPS:+${EXTRA[@]/#/--commands }} "${SIZE_ARGS[@]}" --json cuda.jsonl
    done
    ) |& tee -a cuda.log
done
PYTHONPATH="$here" python -m hpc_patterns_b200.utils.parse cuda.log
