"""Bench line of mate-overlap masking (`--mask-overlaps`, K10p / K10 / K10u; an extension): bench.py's single-GPU
step over BASELINE.json configs[3] (`cfg4_5Mb_200x`, as bench.py builds it), then the new kernels over two workloads
of the same size (synth.simple_pairs):

  pairs      2 x 150 bp mates of ~N(300, 40) bp fragments over one 5 Mb contig at 200x
  amplicon   the mates of whole tiled amplicons (synth.tiled_scheme): one starts in the left primer, one ends in the
             right one

    python tools/bench_mates.py [--steps K] [--warmup W]      # one JSON line on stdout

Per workload (`mates_ms`, medians of 7 alternating rounds of 20 launches): the compaction and torch sort of the
eligible reads, K10p alone (kdl_mates_pair), K10 alone (kdl_overlap_count + kdl_overlap_apply over outputs allocated
once) and K10u (kdl_overlap_untake of the drop rows), against K0 + K1 (the pileup into a reused table).  `parity`: the
masked run's table has the sha256 of an independent restatement -- pairs by fragment number, each R2 base at a cursor
where its R1 has a non-N base read as N by the C quality oracle (oracle/kindel_qoracle.c); these mates have no
indels, so there are no drop rows.  `e2e` times bam_to_consensus(path, mask_overlaps=True) against
bam_to_consensus(path) on a 10^6-read paired BAM, best of 3, alternating; `gpu` is the card's name and power limit,
read in the same run.  Writes nothing into the tree."""
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


def sha(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def restated(batch, frag):
    """The rule for simple, indel-free mates, vectorised: R2's bases at cursors where R1 has a base other than N."""
    from oracle import qoracle

    order = np.argsort(frag, kind="stable")
    a, b = order[0::2], order[1::2]                       # the two reads of every fragment
    r1 = np.where(batch.pair_role[a] == 1, a, b)
    r2 = np.where(batch.pair_role[a] == 1, b, a)
    s1, s2 = batch.ref_start[r1].astype(np.int64), batch.ref_start[r2].astype(np.int64)
    L = batch.seq_len.astype(np.int64)
    lo, hi = np.maximum(s1, s2), np.minimum(s1 + L[r1], s2 + L[r2])
    k = np.maximum(hi - lo, 0)
    qual = np.full(int(L.sum()), 0xFF, dtype=np.uint8)
    base_of = np.concatenate(([0], np.cumsum(L)))[:-1]
    for c0 in range(0, r2.shape[0], 1 << 18):
        sl = slice(c0, c0 + (1 << 18))
        kk = k[sl]
        x = np.repeat(lo[sl], kk) + (np.arange(int(kk.sum())) - np.repeat(np.cumsum(kk) - kk, kk))
        q1 = x - np.repeat(s1[sl], kk)
        w = batch.seq4[np.repeat(batch.seq_off[r1[sl]].astype(np.int64), kk) + (q1 >> 3)]
        nib = (w >> (28 - 4 * (q1 & 7)).astype(np.uint32)) & 0xF
        cov = nib != 15
        q2 = (x - np.repeat(s2[sl], kk))[cov]
        qual[np.repeat(base_of[r2[sl]], kk)[cov] + q2] = 0
    return qoracle.pileup(batch, qual, 1)[0]


def mate_workload(batch, frag, torch, dev):
    from kindel_b200 import _ffi, engine

    lib = _ffi.load()
    st = int(torch.cuda.current_stream(dev).cuda_stream)
    plain = engine.upload(batch, dev)
    table = engine.CountTable(batch.n_slots, dev)
    masked = engine.mask_overlaps(engine.upload(batch, dev))
    got = engine.pileup(masked)[0].cpu().numpy()
    t_hash = torch.from_numpy(batch.name_hash.view(np.int64)).to(dev)
    t_role = torch.from_numpy(batch.pair_role).to(dev)
    t_ms = torch.from_numpy(batch.mate_start).to(dev)
    idx = torch.nonzero(t_role, as_tuple=True)[0]
    order = idx.index_select(0, torch.sort(t_hash.index_select(0, idx), stable=True)[1]).to(torch.int32)
    mate = torch.empty(batch.n_reads, dtype=torch.int32, device=dev)
    n = batch.n_reads
    scratch = torch.empty(int(lib.kdl_overlap_scratch_words(n)), dtype=torch.int32, device=dev)
    mate_ref = engine.pair_mates(masked)
    lib.kdl_overlap_count(C.byref(masked.struct), None, mate_ref.data_ptr(), scratch.data_ptr(), st)
    tot = scratch[-8:].cpu().numpy().view(np.uint32).astype(np.int64)
    out = [torch.empty(max(int(k), 1), dtype=torch.int32, device=dev) for k in (tot[0], tot[0] + 1, tot[1])]
    om = _ffi.KdlQmask(int(tot[0]), int(tot[1]), *(int(x.data_ptr()) for x in out))
    drops = torch.zeros((max(int(tot[2]), 1), 4), dtype=torch.int32, device=dev)

    def sort():
        i = torch.nonzero(t_role, as_tuple=True)[0]
        return i.index_select(0, torch.sort(t_hash.index_select(0, i), stable=True)[1])

    def k10p():
        lib.kdl_mates_pair(C.byref(plain.struct), t_hash.data_ptr(), t_ms.data_ptr(), t_role.data_ptr(),
                           order.data_ptr(), int(order.numel()), mate.data_ptr(), st)

    def k10():
        base = (C.byref(masked.struct), None, mate_ref.data_ptr(), scratch.data_ptr())
        lib.kdl_overlap_count(*base, st)
        lib.kdl_overlap_apply(*base, int(masked.tensors["seq4"].data_ptr()), C.byref(om), drops.data_ptr(),
                              int(tot[2]), st)

    scratch_table = torch.zeros((_ffi.KDL_NCOL, batch.n_slots), dtype=torch.int32, device=dev)
    timing = alternate((("k0_k1_pileup", lambda: engine.pileup(plain, check=False, table=table)),
                        ("compact_sort", sort), ("k10p_pair", k10p), ("k10_overlap", k10),
                        ("k10u_untake", lambda: lib.kdl_overlap_untake(drops.data_ptr(), int(tot[2]),
                                                                       scratch_table.data_ptr(), batch.n_slots, st))),
                       torch)
    again = engine.pileup(masked)[0].cpu().numpy()
    pairs, bases, dels, ins = masked.overlap_masked
    timing.update(reads=int(n), pairs=int(pairs), masked_bases=int(bases), drop_rows=int(dels + ins),
                  note="k10_overlap: the two entry points over preallocated outputs, no read-back; k10p_pair: "
                       "kdl_mates_pair over the sorted order; compact_sort: torch nonzero + sort of the hashes; "
                       "k10u_untake: its drop rows into a scratch table; k0_k1_pileup: engine.pileup, reused table")
    print("mates: timed %d reads, checking against the restatement" % n, file=sys.stderr, flush=True)
    want = restated(batch, frag)
    return timing, {"table_sha256": sha(got), "oracle_sha256": sha(want),
                    "parity": bool(sha(got) == sha(want) == sha(again))}


def e2e(rounds=3):
    from kindel_b200 import kindel as K
    from kindel_b200 import synth

    sub, flag, frag = synth.simple_pairs(4, 750_000, 200)  # 10^6 reads, as bench.py's host block
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "pairs.bam")
        synth.write_paired_bam(path, sub, flag, frag)
        K.bam_to_consensus(path, mask_overlaps=True), K.bam_to_consensus(path)  # warm
        best = {"mates": None, "plain": None}
        for _ in range(rounds):
            for key, fn in (("mates", lambda: K.bam_to_consensus(path, mask_overlaps=True)),
                            ("plain", lambda: K.bam_to_consensus(path))):
                t0 = time.perf_counter()
                fn()
                dt = time.perf_counter() - t0
                best[key] = dt if best[key] is None or dt < best[key] else best[key]
    return {"mates_s": best["mates"], "plain_s": best["plain"], "reads": int(sub.n_reads),
            "note": "bam_to_consensus(path, mask_overlaps=True) vs bam_to_consensus(path), best of %d, alternating"
                    % rounds}


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
    pairs, _, frag = synth.simple_pairs(4, 5_000_000, 200)
    out["pairs"] = mate_workload(pairs, frag, torch, dev)
    del pairs
    torch.cuda.empty_cache()
    rows = synth.tiled_scheme(1, ["ctg0"], [5_000_000])
    amp, _, frag = synth.simple_pairs(5, 5_000_000, 200, amplicons=rows)
    out["amplicon"] = mate_workload(amp, frag, torch, dev)
    del amp
    torch.cuda.empty_cache()
    print("timing bam_to_consensus", file=sys.stderr, flush=True)
    e2e_line = e2e()
    parity = all(v[1]["parity"] for v in out.values())
    ms_per_step = tm["total_ms"] / tm["reps"]
    line = {
        "metric": bench.METRIC, "value": cfg["aligned"] / (ms_per_step * 1e-3), "unit": bench.UNIT,
        "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms_per_step, "higher_is_better": True,
        "dtype": "int32", "data": "synthetic", "steps_timed": tm["reps"], "step_ms": bench.quantiles(tm["step_ms"]),
        "parity": parity, "parity_detail": {k: v[1] for k, v in out.items()},
        "config": {"workload": WORKLOAD, "reads_per_rank": cfg["reads"], "complex_reads_per_rank": cfg["complex"],
                   "aligned_bases_total": cfg["aligned"], "tool": "tools/bench_mates.py",
                   "parity_oracle": "pairs by fragment number, R2 masked where R1 has a non-N base, over "
                                    "oracle/kindel_qoracle.c"},
        "gpu": gpu, "mates_ms": {k: v[0] for k, v in out.items()}, "e2e_mates": e2e_line, "e2e": None,
    }
    print(json.dumps(line))
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
