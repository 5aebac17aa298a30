"""Turn the JSON rows the programs emit (``--json``) into a roofline report.

Every pattern writes rows with device-timed, max-over-ranks numbers; this module adds the
fraction of the relevant roofline — the H100 SXM data-sheet rates: NVLink 450 GB/s per direction per GPU for
communication paths, 989 TFLOP/s dense bf16 for the GEMMs — and renders markdown tables.
``python -m hpc_patterns_b200.utils.report rows.jsonl [...] > REPORT.md``
"""
from __future__ import annotations

import json
import sys
from typing import Dict, Iterable, List

NVLINK_NOMINAL_GBPS = 450.0     # H100 SXM, NVLink 4, per direction (900 GB/s bidirectional), data sheet
BF16_DENSE_TFLOPS = 989.0       # H100 SXM dense bf16 at up to 700 W, data sheet


def load_rows(paths: Iterable[str]) -> List[Dict]:
    rows: List[Dict] = []
    for p in paths:
        with open(p) as f:
            for line in f:
                line = line.strip()
                if line.startswith("{"):
                    try:
                        rows.append(json.loads(line))
                    except json.JSONDecodeError:
                        pass
    return rows


def p2p_table(rows: List[Dict]) -> str:
    out = ["| label | transport | engine | ranks | bytes | uni GB/s | bi GB/s | uni per pair / 450 |",
           "|---|---|---|---|---|---|---|---|"]
    for r in rows:
        if r.get("pattern") != "peer2pear":
            continue
        per_pair = r["uni_GBps"] / max(r["ranks"] // 2, 1)
        out.append(f"| {r.get('label','')} | {r.get('transport','')} | {r.get('engine','')} | {r['ranks']} | "
                   f"{r['bytes']} | {r['uni_GBps']:.1f} | {r['bi_GBps']:.1f} | "
                   f"{per_pair / NVLINK_NOMINAL_GBPS:.2f} |")
    return "\n".join(out)


def allreduce_table(rows: List[Dict]) -> str:
    out = ["| algo | type | ranks | elements | ms | GB/s sent per rank | / 450 |",
           "|---|---|---|---|---|---|---|"]
    for r in rows:
        if r.get("pattern") != "allreduce":
            continue
        g = r["GBps_sent_per_rank"]
        out.append(f"| {r['algo']} | {r['type']} | {r['ranks']} | {r['elements']} | {r['ms']:.4f} | {g:.1f} | "
                   f"{g / NVLINK_NOMINAL_GBPS:.2f} |")
    return "\n".join(out)


def concurency_table(rows: List[Dict]) -> str:
    out = ["| backend | mode | commands | serial us | concurrent us | speedup | max speedup | overlap | verdict |",
           "|---|---|---|---|---|---|---|---|---|"]
    for r in rows:
        if r.get("pattern") != "concurency":
            continue
        out.append(f"| {r['backend']} | {r['mode']} | {' '.join(r['commands'])} | {r['serial_total_us']} | "
                   f"{r['concurrent_total_us']} | {r['speedup']:.2f} | {r['max_speedup']:.2f} | "
                   f"{100 * r['overlap_fraction']:.0f}% | {r['verdict']} |")
    return "\n".join(out)


def tensor_parallel_table(rows: List[Dict]) -> str:
    """Rows of ``python -m hpc_patterns_b200 tp`` (one JSON object per run: ranks, m, n, k and one sub-object per
    layer).  The roofline of a fused layer is the slower of its GEMM at the data-sheet bf16 rate and its bytes over
    NVLink at the nominal 450 GB/s per direction."""
    peak = BF16_DENSE_TFLOPS
    out = ["| layer | ranks | M | N | K | fused ms | stock ms (cuBLAS + NCCL) | speed-up | TFLOP/s per GPU | "
           "roofline ms (tensor / NVLink) | fraction |", "|---|---|---|---|---|---|---|---|---|---|---|"]
    for r in rows:
        if "row_parallel" not in r and "column_parallel" not in r:
            continue
        P, m, n, k = r["ranks"], r["m"], r["n"], r["k"]
        layers = (("row_parallel", 2.0 * m * n * (k // P), m * n * 4 * (P - 1) / P),
                  ("row_parallel_allreduce", 2.0 * m * n * (k // P), m * n * 4 if P > 1 else 0),
                  ("column_parallel", 2.0 * m * (n // P) * k, m * k * 2 * (P - 1) / P))
        for name, flops, link_bytes in layers:
            d = r.get(name)
            if not isinstance(d, dict) or "fused_ms" not in d:
                continue
            t_tensor = flops / (peak * 1e9)
            t_link = link_bytes / (NVLINK_NOMINAL_GBPS * 1e6)
            roof = max(t_tensor, t_link)
            label = name + (f" (chunk {r['chunk']})" if "chunk" in r else "")
            out.append(f"| {label} | {P} | {m} | {n} | {k} | {d['fused_ms']:.4f} | {d['stock_ms']:.4f} | "
                       f"{d['speedup']:.2f} | {flops / d['fused_ms'] / 1e9:.0f} | {t_tensor:.3f} / {t_link:.3f} | "
                       f"{roof / d['fused_ms']:.2f} |")
    return "\n".join(out)


def gemm_table(rows: List[Dict]) -> str:
    """Rows of scripts/gemm_put_bench.py."""
    out = ["| M | N | K | ranks | ours TFLOP/s | cuBLAS | ours / data-sheet peak | fused GEMM->put ms | "
           "stock ms |", "|---|---|---|---|---|---|---|---|---|"]
    for r in rows:
        if "gemm_tflops" not in r:
            continue
        nan = float("nan")
        out.append(f"| {r['m']} | {r['n']} | {r['k']} | {r.get('ranks', 1)} | {r['gemm_tflops']:.0f} | "
                   f"{r['cublas_tflops']:.0f} | {r['gemm_tflops'] / BF16_DENSE_TFLOPS:.2f} | "
                   f"{r.get('fused_gemm_put_ms', nan):.3f} | {r.get('stock_cublas_then_memcpy_ms', nan):.3f} |")
    return "\n".join(out)


def render(rows: List[Dict]) -> str:
    parts = ["# Measured rows (device-timed, max over ranks)\n"]
    if any(r.get("pattern") == "peer2pear" for r in rows):
        parts += ["## peer2pear\n", p2p_table(rows), ""]
    if any(r.get("pattern") == "allreduce" for r in rows):
        parts += ["## allreduce miniapp\n", allreduce_table(rows), ""]
    if any(r.get("pattern") == "concurency" for r in rows):
        parts += ["## concurrency bench\n", concurency_table(rows), ""]
    if any("row_parallel" in r or "column_parallel" in r for r in rows):
        parts += ["## tensor-parallel layers (GEMM fused with its collective)\n", tensor_parallel_table(rows), ""]
    if any("gemm_tflops" in r for r in rows):
        parts += ["## tensor-core GEMM (-> put)\n", gemm_table(rows), ""]
    return "\n".join(parts)


def main(argv=None) -> int:
    argv = list(sys.argv[1:] if argv is None else argv)
    if not argv:
        print("usage: report rows.jsonl [more.jsonl ...]", file=sys.stderr)
        return 2
    print(render(load_rows(argv)))
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
