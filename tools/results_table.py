#!/usr/bin/env python
"""Markdown table of the bench lines kept under profiles/ (one JSON line per file, as bench.py printed it).

    python tools/results_table.py [profiles/h100_bench_*.json ...]      # -> stdout

README.md's results section is this output: regenerate it whenever the files under profiles/ are refreshed, so the
table can never drift from the evidence it cites.
"""
from __future__ import annotations

import glob
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def last_json_line(path: str) -> dict | None:
    try:
        lines = [ln for ln in open(path).read().splitlines() if ln.lstrip().startswith("{")]
        return json.loads(lines[-1])
    except (OSError, IndexError, ValueError):
        return None


def fmt(v: float | None, spec: str = ".3g") -> str:
    return "—" if v is None else format(v, spec)


def row(path: str, d: dict) -> str:
    name = os.path.relpath(path, ROOT)
    if d.get("impl") == "reference":
        cb = d.get("cpu_baseline", {})
        return (f"| `{name}` | reference arm ({cb.get('kind', '?')}, {cb.get('cores', '?')} core) | 1 host | — | "
                f"{fmt(d.get('value'))} | — | — | — | — |")
    cfg = d.get("config", {})
    roof = d.get("roofline") or {}  # (null on a line that does not take the roofline)
    e2e = d.get("e2e") or {}  # (null on an --iupac-threshold line: the host-buffer call has no IUPAC vote)
    km = d.get("kernels_ms", {})
    work = cfg.get("workload", "?")
    cx = cfg.get("complex_reads_per_rank")
    if cx:
        work += f" ({cx} complex reads/GPU)"
    if d.get("iupac_threshold") is not None:
        work += f", IUPAC vote at {d['iupac_threshold']}"
    if d.get("qualities"):
        work += ", + per-base qualities"
    if d.get("variants"):
        work += ", + variant sites (K6)"
    if d.get("variant_ref_ms"):
        work += ", + variants against a reference (K6r, K7)"
    if d.get("strand_ms"):
        work += ", + strand split (K8, reverse pileup)"
    if d.get("primers_ms"):
        work += ", + primer masking (K9, K1q)"
    if d.get("amplicons_ms"):
        work += ", + per-amplicon report (K12, label counts, K12d)"
    if d.get("normalise_ms"):
        work += ", + depth normalisation (K12, K13) at N = %d" % cfg.get("cap", 0)
    if d.get("dedup_ms"):
        work += ", + duplicate removal (K10p, K14k, sort, K14s)"
    if d.get("mates_ms"):
        work += ", + mate-overlap masking (K10p, K10, K10u)"
    if d.get("cohort_ms"):
        work += ", multi-sample VCF (%d samples, K6m)" % cfg.get("samples", 0)
    if d.get("floor"):
        work += ", K11 quality sums alone: %.3f ms, %.2f of its HBM floor" % (km.get("k0_k11_k11g_median", 0),
                                                                           d["floor"].get("share_of_floor", 0))
    if d.get("weights_floor"):
        qv = d.get("quality_vote_ms", {})
        work += ", K11w quality weights alone: %.3f ms, %.2f of its HBM floor; K2w %.3f ms" % (
            qv.get("k0_k11w_median", 0), d["weights_floor"].get("share_of_floor", 0), qv.get("k2w_median", 0))
    if d.get("map_ab"):
        work += ", zeroing A/B (dirty-sector map)"
    out = (f"| `{name}` | {work} | {d.get('n_gpus')} | {fmt(d.get('ms_per_step'), '.4f')} | {fmt(d.get('value'))} | "
           f"{fmt(km.get('k0_k1_pileup'), '.4f')} | {fmt(roof.get('frac'), '.3f')} | {fmt(e2e.get('value'))} | "
           f"{d.get('parity')} |")
    ss = d.get("strong_scaling")
    if ss:
        out += (f"\n| 〃 `strong_scaling` | {ss.get('workload')} cut {d.get('n_gpus')} ways | {d.get('n_gpus')} | "
                f"{fmt(ss.get('ms_per_step'), '.4f')} | {fmt(ss.get('value'))} | {fmt(ss.get('k0_k1_ms'), '.4f')} | — | — | "
                f"{ss.get('parity')} |")
    return out


def main(argv: list[str]) -> int:
    paths = argv or sorted(glob.glob(os.path.join(ROOT, "profiles", "h100_bench_n*.json"))) + \
        sorted(glob.glob(os.path.join(ROOT, "profiles", "h100_bench_reference_arm.json")))
    print("| file | workload | GPUs | ms/step | aligned bases/s (`value`) | K0+K1 ms | roofline frac | e2e bases/s | parity |")
    print("|---|---|---|---|---|---|---|---|---|")
    for p in paths:
        d = last_json_line(p)
        if d is not None:
            print(row(p, d))
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
