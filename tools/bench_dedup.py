"""Bench line of duplicate removal (`--dedup`, K10p + K14k + the sort + K14s; an extension): bench.py's single-GPU step
over BASELINE.json configs[3] (`cfg4_5Mb_200x`, as bench.py builds it), then the dedup device work over two paired
workloads of cfg 4's size (synth.dup_pairs: 2 x 150 bp mates, a fifth of the fragments copied 1-5 more times with fresh
qualities, 5' soft clips and swapped first mates):

  cfg4_shotgun   shotgun pairs over 5 Mb at 200x: ~N(300, 40) bp fragments at random places
  cfg4_amplicon  the same fragments made whole amplicons of synth.tiled_scheme (24 999 amplicons): every fragment of an
                 amplicon has the same two ends, so nearly every pair is a duplicate of thousands

    python tools/bench_dedup.py [--steps K] [--warmup W]      # one JSON line on stdout

On top of bench.py's fields the line carries, per workload (`dedup_ms`):
  `ms`        K10p (engine.pair_mates: the role compaction, the torch sort of name hashes and kdl_mates_pair), K14k
              (kdl_dedup_entries into preallocated lists), the sort (the stable torch.sort passes of both lists) and
              K14s (kdl_dedup_select), against K0 + K1 (the pileup into a reused table) on the same batch, in 7
              alternating rounds of 20 launches; the reads, entries and removals;
  `floor`     the bytes K14k and K14s must move, counted from the shapes below, and the time they would take at the data
              sheet's 3.35 TB/s -- a lower bound, not a rate reached;
  `parity`    the keep bytes and the totals equal oracle/py_doracle.py's keep_vectorised over the batch's ends and the
              fragments' own pairing (sha256 of both).
`e2e_dedup` times bam_to_consensus(path, dedup=True) against bam_to_consensus(path) on a 10^6-read paired BAM, best of
3, alternating; `gpu` is the card's name and power limit, read in the same run.  bench.py's step runs none of this.
Writes nothing into the tree."""
from __future__ import annotations

import argparse
import ctypes as C
import hashlib
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from bench_fastq import alternate  # noqa: E402
from bench_variants_ref import gpu_info  # noqa: E402

WORKLOAD = "cfg4_5Mb_200x"
HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def sha(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def oracle_inputs(b, frag):
    """(u, left alone, mate) of dup_pairs' reads (one M op, or an M op and a 5' soft clip): the oracle's own ends and
    the pairing by fragment (R2 -> R1, neither KDL_HARD)."""
    co = b.cig_off.astype(np.int64)
    first, last = b.cigar[co[:-1]], b.cigar[co[1:] - 1]
    lead = np.where((first & 15) == 4, first >> 4, 0).astype(np.int64)
    trail = np.where(((last & 15) == 4) & (co[1:] - co[:-1] > 1), last >> 4, 0).astype(np.int64)
    start = b.ref_start.astype(np.int64)
    u = np.where(b.reverse == 1, start + (b.seq_len - lead - trail) - 1 + trail, start - lead)
    order = np.argsort(frag, kind="stable")
    a, c = order[0::2], order[1::2]
    r1, r2 = np.where(b.pair_role[a] == 1, a, c), np.where(b.pair_role[a] == 1, c, a)
    hard = (b.l_seq.view(np.uint32) & 0x40000000) != 0
    ok = ~hard[r1] & ~hard[r2]
    mate = np.full(b.n_reads, -1, dtype=np.int64)
    mate[r2[ok]] = r1[ok]
    return u, b.dup_score < 0, mate


def floor_bytes(n, n_complex, ops_complex, n_pair, n_single):
    """Bytes K14k and K14s read and write at least once each, from the shapes: K14k-e reads l_seq, ref_start, seq_off,
    reverse, score (17 B per read) and a complex read's two header words and ops, writes end, keep, paired (10 B);
    K14k-p and K14k-s read mate, end and paired again (13 B per read) and write a pair entry (36 B) with its two
    markers (2 x 24 B) or a single (24 B); K14s per entry reads the order (8 B), the key of it and of the one before
    (pair 20 B, single 12 B, twice: K14s-h and K14s-b), the rank (8 B, twice) and writes best (8 B), run (4 B, read
    back), keep where removed (ignored)."""
    k14k = n * (17 + 10 + 13) + 4 * (2 * n_complex + ops_complex) + n_pair * (36 + 48) + (n_single - 2 * n_pair) * 24
    k14s = n_pair * (8 + 2 * 2 * 20 + 2 * 8 + 8 + 4 + 4) + n_single * (8 + 2 * 2 * 12 + 2 * 8 + 8 + 4 + 4)
    return int(k14k), int(k14s)


def dedup_workload(batch, frag, torch, dev):
    from kindel_b200 import _ffi, engine
    from oracle import py_doracle

    lib = _ffi.load()
    db = engine.upload(batch, dev)
    table = engine.CountTable(batch.n_slots, dev)
    keep, stats = engine.dedup(db)
    st = int(torch.cuda.current_stream(dev).cuda_stream)
    n = int(batch.n_reads)
    mate = engine.pair_mates(db)
    reverse = torch.from_numpy(batch.reverse).to(dev)
    score = torch.from_numpy(batch.dup_score).to(dev)
    t = {f: torch.empty(max(n if full else n // 2, 1), dtype=dt, device=dev) for f, dt, full in engine._DEDUP_LISTS}
    lists = _ffi.KdlDedupLists(*(int(t[f].data_ptr()) for f, _, _ in engine._DEDUP_LISTS))
    keep_buf = torch.empty(max(n, 1), dtype=torch.uint8, device=dev)
    totals = torch.zeros(_ffi.KDL_DEDUP_TOTALS, dtype=torch.int64, device=dev)

    def k14k():
        lib.kdl_dedup_entries(C.byref(db.struct), reverse.data_ptr(), score.data_ptr(), mate.data_ptr(),
                              C.byref(lists), keep_buf.data_ptr(), totals.data_ptr(), st)

    k14k()
    n_pair, n_single = (int(x) for x in totals[:2].cpu())
    pk = [t["pair_e1"][:n_pair], t["pair_e2"][:n_pair]]
    sk = [t["single_key"][:n_single]]
    orders = {}

    def sort():
        orders["p"] = engine._lexsort(pk)
        orders["s"] = engine._lexsort(sk)

    sort()
    words = int(lib.kdl_dedup_scratch_words(max(n_pair, n_single)))
    scratch = torch.empty(max(words, 2), dtype=torch.int32, device=dev)

    def k14s():
        lib.kdl_dedup_select(C.byref(lists), orders["p"].data_ptr(), n_pair, orders["s"].data_ptr(), n_single,
                             scratch.data_ptr(), words, keep_buf.data_ptr(), totals.data_ptr(), st)

    k14k()
    sort()
    k14s()
    same = bool(torch.equal(keep_buf[:n], keep))
    timing = alternate((("k0_k1_pileup", lambda: engine.pileup(db, check=False, table=table)),
                        ("k10p_pair", lambda: engine.pair_mates(db)), ("k14k_entries", k14k), ("sort", sort),
                        ("k14s_select", k14s)), torch)
    co = batch.cig_off.astype(np.int64)
    cx = batch.complex_idx.astype(np.int64)
    b_k, b_s = floor_bytes(n, int(batch.n_complex), int((co[cx + 1] - co[cx]).sum()), n_pair, n_single)
    timing.update(reads=n, complex=int(batch.n_complex), pair_entries=n_pair, single_list_entries=n_single,
                  pairs_removed=stats[0], singles_removed=stats[1], shadowed=stats[2],
                  floor={"k14k_bytes": b_k, "k14s_bytes": b_s, "k14k_ms_at_3.35TBps": 1e3 * b_k / HBM_BYTES_PER_S,
                         "k14s_ms_at_3.35TBps": 1e3 * b_s / HBM_BYTES_PER_S},
                  note="k10p_pair: engine.pair_mates (role compaction, torch sort of the name hashes, kdl_mates_pair); "
                       "k14k_entries: kdl_dedup_entries into preallocated lists; sort: the stable torch.sort passes "
                       "of both lists (one contig: no contig pass); k14s_select: kdl_dedup_select; k0_k1_pileup: "
                       "engine.pileup into a reused CountTable")
    print("dedup: timed %d reads, checking against the oracle" % n, file=sys.stderr, flush=True)
    u, alone, omate = oracle_inputs(batch, frag)
    want, wt = py_doracle.keep_vectorised(np.zeros(n, dtype=np.int64), u, batch.reverse, alone, batch.dup_score, omate)
    got = keep.cpu().numpy()
    detail = {"keep_sha256": sha(got), "oracle_keep_sha256": sha(want), "totals": list(stats),
              "oracle_totals": list(wt)}
    detail["parity"] = bool(sha(got) == sha(want) and tuple(stats) == tuple(wt) and same)
    return timing, detail


def e2e(rounds=3):
    from kindel_b200 import kindel as K
    from kindel_b200 import synth

    b, flag, frag, qual = synth.dup_pairs(4, 750_000, 200, clip_frac=0.0, want_qual=True)  # 10^6 reads
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "pairs.bam")
        synth.write_simple_bam(path, b, names=synth.pair_names(frag), flag=flag, next_pos=b.mate_start, qual=qual)
        on = lambda: K.bam_to_consensus(path, dedup=True)  # noqa: E731
        off = lambda: K.bam_to_consensus(path)  # noqa: E731
        on(), off()  # warm
        best = {"dedup": None, "default": None}
        for _ in range(rounds):
            for key, fn in (("dedup", on), ("default", off)):
                t0 = time.perf_counter()
                fn()
                dt = time.perf_counter() - t0
                best[key] = dt if best[key] is None or dt < best[key] else best[key]
        run = K.pileup_run(path, dedup=True)[0]
    return {"consensus_dedup_s": best["dedup"], "consensus_s": best["default"], "reads": int(b.n_reads),
            "deduplicated": list(run.deduplicated),
            "note": "bam_to_consensus(path, dedup=True) vs bam_to_consensus(path), best of %d, alternating" % rounds}


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args(argv)

    import torch

    from kindel_b200 import engine, synth

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    gpu = gpu_info()
    batch = bench.gen_reads(WORKLOAD)
    db = engine.upload(batch, dev)
    table = engine.CountTable(batch.n_slots, dev)
    calls_buf = torch.empty(batch.n_slots, dtype=torch.uint8, device=dev)

    def step(timers=None):
        if timers:
            timers[0].record()
        engine.pileup(db, check=False, table=table)
        if timers:
            timers[1].record()
        out = engine.vote(table.t, 1, out=calls_buf)
        if timers:
            timers[2].record()
        return out

    tm = bench.time_steps(step, args.steps, args.warmup, torch, None, 1, dev)
    cfg = dict(reads=int(batch.n_reads), complex=int(batch.n_complex), aligned=int(batch.aligned_bases))
    del db, table, batch
    torch.cuda.empty_cache()
    print("step timed: %.4f ms" % (tm["total_ms"] / tm["reps"]), file=sys.stderr, flush=True)
    out = {}
    for name, amplicons in (("cfg4_shotgun", None), ("cfg4_amplicon", synth.tiled_scheme(4, ["ctg0"], [5_000_000]))):
        b, flag, frag, _ = synth.dup_pairs(4, 5_000_000, 200, amplicons=amplicons)
        out[name] = dedup_workload(b, frag, torch, dev)
        del b
        torch.cuda.empty_cache()
    print("timing bam_to_consensus with dedup", file=sys.stderr, flush=True)
    e2e_line = e2e()
    parity = all(v[1]["parity"] for v in out.values())
    ms_per_step = tm["total_ms"] / tm["reps"]
    line = {
        "metric": bench.METRIC, "value": cfg["aligned"] / (ms_per_step * 1e-3), "unit": bench.UNIT,
        "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms_per_step, "higher_is_better": True,
        "dtype": "int32", "data": "synthetic", "steps_timed": tm["reps"], "step_ms": bench.quantiles(tm["step_ms"]),
        "parity": parity, "parity_detail": {k: v[1] for k, v in out.items()},
        "config": {"workload": WORKLOAD, "reads_per_rank": cfg["reads"], "complex_reads_per_rank": cfg["complex"],
                   "aligned_bases_total": cfg["aligned"], "tool": "tools/bench_dedup.py",
                   "parity_oracle": "oracle/py_doracle.py (keep_vectorised, pairs by fragment)"},
        "gpu": gpu, "dedup_ms": {k: v[0] for k, v in out.items()}, "e2e_dedup": e2e_line, "e2e": None,
    }
    print(json.dumps(line))
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
