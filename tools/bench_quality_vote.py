"""Bench line of the quality vote (an extension, `consensus --quality-vote`): BASELINE.json configs[3] (`cfg4_5Mb_200x`,
as bench.py builds it) with the seeded qualities of synth.qualities.

    python tools/bench_quality_vote.py [--rounds R] [--out FILE]     # one JSON line on stdout (and in FILE)

Reports, on one GPU:
  * K0 + K11w (kdl_quality_weights) against K0 + K11 (kdl_quality_pileup), and K2w (kdl_vote_quality, with its Q
    bytes) against K2 (kdl_vote), each the median of R alternating rounds timed with CUDA events, and K11w's share of
    its floor: the bytes it must move -- seq4 and qual8 read, wsum written -- over the data sheet's 3.35 TB/s;
  * `parity`: the sha256 of wsum, the calls and their Q against a restatement that never reads the engine (numpy per
    chunk of simple reads, oracle/py_qvoracle.py's walk over weights for the complex ones, the vote in numpy over the
    pileup's table);
  * on a 10^6-read BAM written with qualities, bam_to_consensus(quality_vote=True) against the default, wall clock,
    best of 3, alternating.
The card's name and power limit are read in the same run.  The default FILE is
profiles/h100_bench_n1_cfg4_5Mb_200x_quality_vote.json."""
from __future__ import annotations

import argparse
import ctypes as C
import hashlib
import json
import os
import statistics
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (the workload generator and clock sampler of the main bench)

WORKLOAD = "cfg4_5Mb_200x"
HBM_TBPS = 3.35


def oracle_weights(batch, qual):
    """wsum uint64 [4, n_slots] without the engine: simple reads in numpy chunks (one M op at contig_slot +
    ref_start), complex reads through py_qvoracle.walk with every quality replaced by its weight."""
    from kindel_b200.quality import WEIGHT
    from oracle import py_oracle, py_qvoracle

    wt = np.array(WEIGHT, dtype=np.int64)
    n_slots = int(batch.n_slots)
    wsum = np.zeros((4, n_slots), dtype=np.uint64)
    lens = batch.seq_len.astype(np.int64)
    qoff = np.concatenate(([0], np.cumsum(lens)))
    contig = np.repeat(np.arange(batch.n_contigs), np.diff(batch.contig_read_off))
    start = batch.contig_slot[contig].astype(np.int64) + batch.ref_start.astype(np.int64)
    simple = (batch.l_seq.astype(np.int64) & 0x80000000) == 0
    shifts = np.arange(28, -4, -4, dtype=np.uint32)
    step = 200_000
    for r0 in range(0, batch.n_reads, step):
        idx = np.flatnonzero(simple[r0:r0 + step]) + r0
        if idx.size == 0:
            continue
        ln = lens[idx]
        k = np.arange(int(ln.sum()), dtype=np.int64) - np.repeat(np.cumsum(ln) - ln, ln)
        rr = np.repeat(idx, ln)
        w = batch.seq4[batch.seq_off[rr].astype(np.int64) + (k >> 3)]
        nib = (w >> shifts[k & 7]) & 15
        q = wt[np.minimum(qual[qoff[rr] + k].astype(np.int64), 93)]
        slot = start[rr] + k
        for col, v in enumerate((1, 2, 4, 8)):
            m = nib == v
            # (float64 sums of integers below 2^53 are exact)
            wsum[col] += np.bincount(slot[m], weights=q[m].astype(np.float64), minlength=n_slots).astype(np.uint64)
    recs = py_oracle.records_of(batch)

    class Sparse(dict):  # a per-read accumulator that walk() can += into like a list
        def __missing__(self, key):
            return 0

    for r in np.flatnonzero(~simple).tolist():
        c = int(contig[r])
        L, s0 = int(batch.contig_len[c]), int(batch.contig_slot[c])
        q4 = [Sparse() for _ in range(4)]
        py_qvoracle.walk(L, recs[r], [WEIGHT[min(x, 93)] for x in qual[qoff[r]:qoff[r + 1]].tolist()], set(), q4,
                         Sparse())
        for col in range(4):
            for p, v in q4[col].items():
                wsum[col, s0 + p] += np.uint64(v)
    return wsum


def oracle_vote(counts, wsum, min_depth_ceil=1):
    """(calls, qual) uint8 of the quality vote in numpy: consensus_sequence's D / N / I decisions (kindel.py:402-424)
    over the count table, the base with the largest weight sum (N on a tie or at zero), Q = min(60, gap >> 16)."""
    c = counts[0:7].astype(np.int64)
    depth = c[0:4].sum(axis=0)
    dn = np.concatenate((depth[1:], [0]))
    change = np.where(2 * c[6] > np.minimum(depth, dn), 3, 0)
    order = np.sort(wsum, axis=0)
    best, second = order[3], order[2]
    b = np.argmax(wsum, axis=0)
    none = (best == 0) | (best == second)
    base = np.where(none, 4, b)
    q = np.where(none, 0, np.minimum((best - second) >> np.uint64(16), 60)).astype(np.uint8)
    calls = ((change << 4) | base).astype(np.uint8)
    low = depth < min_depth_ceil
    dele = 2 * c[5] > depth
    calls[low], q[low] = (2 << 4) | 4, 0
    calls[dele], q[dele] = (1 << 4) | 4, 0
    return calls, q


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_bench_n1_cfg4_5Mb_200x_quality_vote.json"))
    ap.add_argument("--no-host", action="store_true", help="skip the end-to-end consensus timing")
    args = ap.parse_args(argv)

    import torch

    from kindel_b200 import _ffi, bamio, engine, synth
    from kindel_b200 import kindel as K

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    lib = _ffi.load()
    sampler = bench.ClockSampler(0)
    sampler.start()
    batch = bench.gen_reads(WORKLOAD)
    qual = synth.qualities(7, batch.seq_len)
    qual8 = bamio.qual_layout(batch, qual)
    n_slots = int(batch.n_slots)
    db = engine.upload(batch, dev)
    counts, _ = engine.pileup(db)
    q8 = torch.from_numpy(qual8).to(dev)
    qsum = torch.empty((4, n_slots), dtype=torch.int32, device=dev)
    emass = torch.empty(n_slots, dtype=torch.int64, device=dev)
    wsum = torch.empty((4, n_slots), dtype=torch.int64, device=dev)
    calls = torch.empty(n_slots, dtype=torch.uint8, device=dev)
    qv = torch.empty(n_slots, dtype=torch.uint8, device=dev)
    stream = engine._stream_ptr(dev)

    def k11w():
        _ffi.check(lib.kdl_quality_weights(C.byref(db.struct), q8.data_ptr(), wsum.data_ptr(), n_slots, stream),
                   "kdl_quality_weights")

    def k11():
        _ffi.check(lib.kdl_quality_pileup(C.byref(db.struct), q8.data_ptr(), qsum.data_ptr(), emass.data_ptr(), n_slots,
                                          stream), "kdl_quality_pileup")

    def k2w():
        _ffi.check(lib.kdl_vote_quality(counts.data_ptr(), wsum.data_ptr(), n_slots, 1, calls.data_ptr(), qv.data_ptr(),
                                        stream), "kdl_vote_quality")

    def k2():
        _ffi.check(lib.kdl_vote(counts.data_ptr(), n_slots, 1, calls.data_ptr(), stream), "kdl_vote")

    def timed(fn):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        fn()
        ev[1].record()
        ev[1].synchronize()
        return ev[0].elapsed_time(ev[1])

    for _ in range(3):
        k11w()
        k11()
        k2w()
        k2()
    torch.cuda.synchronize()
    sampler.wait_first_sample()
    sampler.mark()
    t = {"k11w": [], "k11": [], "k2w": [], "k2": []}
    for _ in range(args.rounds):
        for name, fn in (("k11w", k11w), ("k11", k11), ("k2w", k2w), ("k2", k2)):
            t[name].append(timed(fn))
    clocks = sampler.stop()
    k11w()
    k2w()
    torch.cuda.synchronize()
    got_w = wsum.cpu().numpy().view(np.uint64)
    got_c, got_q = calls.cpu().numpy(), qv.cpu().numpy()
    want_w = oracle_weights(batch, qual)
    want_c, want_q = oracle_vote(counts.cpu().numpy(), want_w)
    sha = lambda *a: hashlib.sha256(b"".join(np.ascontiguousarray(x).tobytes() for x in a)).hexdigest()
    got, want = sha(got_w, got_c, got_q), sha(want_w, want_c, want_q)

    floor_bytes = 4 * int(batch.seq4.shape[0]) + qual8.nbytes + 32 * n_slots
    floor_ms = floor_bytes / (HBM_TBPS * 1e12) * 1e3
    med = {k: statistics.median(v) for k, v in t.items()}
    line = {
        "metric": "K11w quality weights and K2w quality vote", "data": "synthetic", "n_gpus": 1,
        "config": {"workload": WORKLOAD + "_quality_vote", "reads": int(batch.n_reads),
                   "complex_reads": int(batch.n_complex), "hard_reads": int(batch.n_hard),
                   "aligned_bases": int(batch.aligned_bases), "tool": "tools/bench_quality_vote.py",
                   "rounds": args.rounds},
        "parity": got == want, "sha256": got,
        "parity_oracle": "numpy over the simple reads + oracle/py_qvoracle.py's walk over weights for the complex "
                         "reads; the vote in numpy over the pileup's table",
        "quality_vote_ms": {"k0_k11w_median": med["k11w"], "k0_k11_median": med["k11"], "k2w_median": med["k2w"],
                            "k2_median": med["k2"], "k11w_min": min(t["k11w"]), "k11w_max": max(t["k11w"])},
        "weights_floor": {"bytes": floor_bytes, "hbm_tbps_datasheet": HBM_TBPS, "ms": floor_ms,
                          "share_of_floor": floor_ms / med["k11w"]},
        "clocks": clocks,
        "gpu": {"name": torch.cuda.get_device_name(dev), "count": 1,
                "power_limit_w": clocks.get("power_limit_w") if clocks else None},
    }
    del db, counts, q8, qsum, emass, wsum, calls, qv
    torch.cuda.empty_cache()
    if not args.no_host:
        sub = synth.simple_reads(9, [5_000_000], 30)
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "q.bam")
            synth.write_simple_bam(path, sub, qual=synth.qualities(9, sub.seq_len))
            ts = {False: [], True: []}
            for _ in range(3):
                for on in (False, True):
                    t0 = time.perf_counter()
                    K.bam_to_consensus(path, quality_vote=on)
                    ts[on].append(time.perf_counter() - t0)
            line["consensus_1e6_reads"] = {"reads": int(sub.n_reads), "ms_default": min(ts[False]) * 1e3,
                                           "ms_quality_vote": min(ts[True]) * 1e3}
    text = json.dumps(line)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(text + "\n")
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
