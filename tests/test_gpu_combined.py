"""The extensions together on the GPU: base / read filters, the IUPAC vote and per-base qualities end to end against
the composed oracle of tests/combo_cases.py; the combined REPORT line by line; the CLI with every option; the launch
count of each extension; the IUPAC exchange (K2x) over masked shards on one GPU; and the reuse of the host-buffer
context's and a CountTable's count table across batches of every kind."""
import ctypes as C

import numpy as np
import pytest

import combo_cases as CC
from kindel_b200 import _ffi, bamio, cli, synth
from kindel_b200 import distributed as D
from kindel_b200 import kindel as K
from oracle import coracle, fqoracle, ioracle, qoracle
from test_combined import SEEDS, _same_as_oracle

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    d = tmp_path_factory.mktemp("combo")
    out = {}
    for seed in SEEDS:
        contigs, recs = CC.combo_case(seed)
        out[seed] = (contigs, recs, CC.write_bam(d / ("c%d.bam" % seed), contigs, recs), d)
    return out


def test_end_to_end_equals_composed_oracle(corpus):
    """bam_to_consensus over the option matrix: sequence, changes and qualities are the composed oracle's; qualities on
    or off, the sequence, changes and REPORT are the same, and the REPORT is the host code's over the oracle's masked
    tables."""
    n_iupac = 0
    for k, (t, bq, md, realign, trim, upper, (mq, ex)) in enumerate(CC.option_matrix()):
        seed = SEEDS[k % len(SEEDS)]
        contigs, recs, path, d = corpus[seed]
        kw = dict(realign=realign, min_depth=md, trim_ends=trim, uppercase=upper, min_base_quality=bq, min_mapq=mq,
                  exclude_flags=ex, iupac_threshold=t)
        what = (seed, kw)
        got = K.bam_to_consensus(path, qualities=True, **kw)
        piled = CC.Piled(contigs, recs, d / "oracle.bam", bq, mq, ex)
        _same_as_oracle(got, piled.consensus(t, md, realign, trim, upper), what)
        plain = K.bam_to_consensus(path, **kw)
        assert [r.sequence for r in plain.consensuses] == [r.sequence for r in got.consensuses], what
        assert all(r.qualities is None for r in plain.consensuses)
        assert plain.refs_changes == got.refs_changes and plain.refs_reports == got.refs_reports, what
        masked = bamio.read_alignment(path, min_mapq=mq, exclude_flags=ex, min_base_quality=bq)
        run = K.PileupRun.from_host_tables(masked, piled.counts, coracle.derive(piled.counts), piled.events)
        host = K.consensus_from_run(run, piled.calls(t, md), path, realign, md, 9, 0.1, 50, trim, upper,
                                    filters=(bq, mq, ex), iupac_threshold=t)
        assert got.refs_reports == host.refs_reports, what
        n_iupac += sum(len(c.iupac) for c in got.refs_changes.values())
    assert n_iupac > 20


def _sites(changes, code):
    return ", ".join(str(k + 1) for k, c in enumerate(changes) if c == code)


def test_combined_report_line_by_line(corpus):
    contigs, recs, path, d = corpus[SEEDS[0]]
    res = K.bam_to_consensus(path, min_base_quality=20, min_mapq=10, exclude_flags=0x400, iupac_threshold=0.6,
                             qualities=True)
    piled = CC.Piled(contigs, recs, d / "oracle.bam", 20, 10, 0x400)
    plain = CC.Piled(contigs, recs, d / "plain.bam", 0, 10, 0x400)
    calls = piled.calls(0.6)
    n_depth_differs = 0
    for c, name, s0, L, _ in piled.contigs():
        acgt = piled.counts[0:4, s0:s0 + L].sum(axis=0)
        n_depth_differs += int(acgt.max() != plain.counts[0:4, s0:s0 + L].sum(axis=0).max())
        changes = res.refs_changes[name]
        iupac = ", ".join(str(k + 1) for k in np.flatnonzero(calls[s0:s0 + L] & 0x80).tolist())
        assert res.refs_reports[name].splitlines() == [
            "========================= REPORT ===========================",
            "reference: %s" % name,
            "options:",
            "- bam_path: %s" % path,
            "- min_depth: 1",
            "- realign: False",
            "    - min_overlap: 9",
            "    - clip_decay_threshold: 0.1",
            "- trim_ends: False",
            "- uppercase: False",
            "- min_base_quality: 20",
            "- min_mapq: 10",
            "- exclude_flags: 0x400",
            "- iupac_threshold: 0.6",
            "observations:",
            "- min, max observed depth: %d, %d" % (acgt.min(), acgt.max()),  # of the masked table
            "- ambiguous sites: " + _sites(changes, "N"),
            "- iupac sites: " + iupac,
            "- insertion sites: " + _sites(changes, "I"),
            "- deletion sites: " + _sites(changes, "D"),
            "- clip-dominant regions: ",
        ], name
    assert n_depth_differs > 0


def test_cli_fastq_with_every_option(corpus, capsys):
    """`consensus --fastq` with the IUPAC vote, all three filters, -r, -t and -u: each FASTQ sequence is the FASTA's of
    the same command without --fastq, byte for byte, stderr is the same, and the qualities are the composed oracle's."""
    contigs, recs, path, d = corpus[SEEDS[1]]
    args = ["consensus", "--iupac-threshold", "0.6", "--min-base-quality", "20", "--min-mapq", "10", "--exclude-flags",
            "0x400", "-r", "-t", "-u", path]
    capsys.readouterr()
    assert cli.main(args) == 0
    fa = capsys.readouterr()
    assert cli.main(args[:1] + ["--fastq"] + args[1:]) == 0
    fq = capsys.readouterr()
    assert fq.err == fa.err and "- min_base_quality: 20" in fq.err and "- iupac_threshold: 0.6" in fq.err
    want = CC.Piled(contigs, recs, d / "oracle.bam", 20, 10, 0x400).consensus(0.6, 1, True, True, True, min_overlap=7)
    lines, fasta = fq.out.split("\n"), fa.out.split("\n")
    assert len(lines) == 4 * len(want) + 1 and len(fasta) == 2 * len(want) + 1
    for r, (name, seq, _, qual) in enumerate(want):
        assert lines[4 * r: 4 * r + 4] == ["@%s_cns" % name, fasta[2 * r + 1], "+", qual]
        assert fasta[2 * r: 2 * r + 2] == [">%s_cns" % name, seq]


def test_launch_counts(corpus):
    """Masking with masked bases adds K1q, filters that mask nothing add nothing, the IUPAC vote adds nothing, qualities
    add K2q + K5q (K2q alone with --realign)."""
    lib = _ffi.load()
    path = corpus[SEEDS[0]][2]

    def launches(**kw):
        K.bam_to_consensus(path, **kw)  # warm
        n0 = lib.kdl_launch_count()
        K.bam_to_consensus(path, **kw)
        return lib.kdl_launch_count() - n0

    base = launches()
    assert min(min(q) for *_, q in corpus[SEEDS[0]][1] if q is not None) >= 2
    assert launches(min_base_quality=2, exclude_flags=0x800) == base  # no base below Q2, no record with 0x800
    assert launches(min_base_quality=20) == base + 1
    assert launches(iupac_threshold=0.6) == base
    assert launches(min_base_quality=20, iupac_threshold=0.6, qualities=True) == base + 3
    real = launches(realign=True)
    assert launches(realign=True, min_base_quality=20, iupac_threshold=0.99, qualities=True) == real + 2


def test_iupac_exchange_over_masked_shards_on_one_gpu(corpus):
    """K2x with the IUPAC vote (kdl_exchange_vote_iupac) for 3 ranks emulated in one process on one GPU, over shards that
    carry their own mask lists: every shard runs K1 + K1q into a reused CountTable bounded by its footprint, twice.
    Every rank's call bytes equal the IUPAC vote of the composed oracle's full masked table at each threshold and
    min_depth, and K2q over K2p's reduced table and the gathered calls equals the oracle's qualities.  The kernels are
    issued signal, vote, wait for all ranks in turn, so no kernel ever waits for a flag that is not already set."""
    import torch

    from kindel_b200 import engine

    lib = _ffi.load()
    dev = torch.device("cuda", torch.cuda.current_device())
    st = int(torch.cuda.current_stream(dev).cuda_stream)
    world = 3
    contigs, recs, path, d = corpus[SEEDS[0]]
    full = bamio.read_alignment(path, min_mapq=10, exclude_flags=0x400, min_base_quality=20)
    piled = CC.Piled(contigs, recs, d / "oracle.bam", 20, 10, 0x400)
    S = full.n_slots
    shards = [D.shard_batch(full, r, world) for r in range(world)]
    assert all(s.n_masked > 0 for s in shards) and sum(s.n_masked for s in shards) == full.n_masked
    feet = [D.footprint(s) for s in shards]
    slices = D.owner_slices(S, world)
    table_bytes, calls_off, flags_off = 19 * S * 4, 19 * S * 4, 19 * S * 4 + S
    blocks = [torch.zeros(flags_off + 256, dtype=torch.uint8, device=dev) for _ in range(world)]
    xs = []
    for r in range(world):
        x = _ffi.KdlExchange()
        x.n_ranks, x.rank = world, r
        for p, blk in enumerate(blocks):
            base = blk.data_ptr()
            x.tables[p], x.calls[p] = base, base + calls_off
            x.ready[p], x.done[p] = base + flags_off, base + flags_off + 64
            x.foot_lo[p], x.foot_hi[p] = feet[p]
            x.slice_lo[p], x.slice_hi[p] = slices[p]
        x.counter = blocks[r].data_ptr() + flags_off + 128
        xs.append(x)
    tables = [blk[:table_bytes].view(torch.int32).view(19, S) for blk in blocks]
    counts = [engine.CountTable(S, dev, tensor=tables[r]) for r in range(world)]
    ptrs = (C.c_void_p * world)(*[blk.data_ptr() for blk in blocks])
    flo = (C.c_int64 * world)(*[f[0] for f in feet])
    fhi = (C.c_int64 * world)(*[f[1] for f in feet])
    epoch = 0
    n_codes = 0
    for step in range(2):  # the second pass reuses the tables (lazy zeroing) and the flags
        for r in range(world):
            engine.pileup(engine.upload(shards[r], dev), check=False, table=counts[r], slot_range=feet[r])
        torch.cuda.synchronize()
        assert np.array_equal(sum(t.cpu().numpy().astype(np.int64) for t in tables), piled.counts)
        for t in (0.0, 0.6, 0.99, 1.0):
            for md in (1, 3):
                epoch += 1
                for r in range(world):
                    _ffi.check(lib.kdl_exchange_signal(C.byref(xs[r]), epoch, st), "signal")
                for r in range(world):
                    _ffi.check(lib.kdl_exchange_vote_iupac(C.byref(xs[r]), S, md, t, epoch, st), "vote")
                for r in range(world):
                    _ffi.check(lib.kdl_exchange_wait(C.byref(xs[r]), epoch, st), "wait")
                torch.cuda.synchronize()
                want = ioracle.vote_iupac(piled.counts, md, t)
                n_codes += int(np.count_nonzero(want & 0x80))
                for r in range(world):
                    got = blocks[r][calls_off:calls_off + S].cpu().numpy()
                    np.testing.assert_array_equal(got, want, err_msg="step %d t %s md %d rank %d" % (step, t, md, r))
                # K2q over K2p's reduced vote columns and the gathered calls
                reduced = torch.zeros((7, S), dtype=torch.int32, device=dev)
                k2p = torch.zeros(S, dtype=torch.uint8, device=dev)
                _ffi.check(lib.kdl_vote_peers_sparse(ptrs, flo, fhi, world, S, 0, S, md, k2p.data_ptr(),
                                                     reduced.data_ptr(), st), "vote_peers")
                q = engine.consensus_qual(reduced, blocks[1][calls_off:calls_off + S]).cpu().numpy()
                np.testing.assert_array_equal(reduced.cpu().numpy(), piled.counts[:7])
                np.testing.assert_array_equal(q, fqoracle.qual(piled.counts, want))
    assert n_codes > 50


def _reuse_sequence(tmp_path):
    """Batches on one contig layout, as (batch, counts, events) with the oracle's tables (None: the batch raises
    IndexError): masked complex, plain simple, masked simple, plain complex twice, a batch that raises, masked
    complex."""
    L = 20_000

    def masked(b, seed):
        m, qual = synth.with_qualities(b, seed)
        assert m.n_masked > 0
        return (m,) + qoracle.pileup(b, qual, 20)

    def plain(b):
        return (b,) + coracle.pileup(b)

    bad = tmp_path / "bad.sam"
    bad.write_text("@SQ\tSN:c0\tLN:%d\n" % L + "".join(
        "r%d\t0\tc0\t%d\t60\t50M\t*\t0\t0\t%s\t*\n" % (k, p, "ACGTA" * 10) for k, p in enumerate([1, 500, L - 10])))
    seq = [masked(synth.complex_reads(31, L, 60), 1), plain(synth.simple_reads(32, [L], 40)),
           masked(synth.simple_reads(33, [L], 40), 2), plain(synth.complex_reads(34, L, 30)),
           plain(synth.complex_reads(35, L, 50)), (bamio.read_alignment(bad), None, None),
           masked(synth.complex_reads(36, L, 40), 3)]
    assert len({b.n_slots for b, _, _ in seq}) == 1
    assert [b.n_complex > 0 for b, _, _ in seq] == [True, False, False, True, True, True, True]
    return seq


def test_host_context_reuses_its_table_across_batch_kinds(tmp_path):
    """One HostContext, one n_slots: every call after the first takes the reuse branch (fresh weights, and the other
    columns zeroed when the previous call had complex reads).  Every call's counts, events and calls equal a fresh
    oracle result; then the same through engine.pileup into one CountTable."""
    import torch

    from kindel_b200 import engine

    seq = _reuse_sequence(tmp_path)
    ctx = engine.HostContext(0)
    try:
        for k, (b, want, want_ev) in enumerate(seq):
            if want is None:
                with pytest.raises(IndexError):
                    ctx.consensus(b, 1)
                continue
            counts = np.full((19, b.n_slots), -1, dtype=np.int32)
            events = np.full((max(b.n_events, 1), 4), -1, dtype=np.int32)
            calls = ctx.consensus(b, 1, counts_out=counts, events_out=events)
            np.testing.assert_array_equal(counts, want, err_msg="call %d" % k)
            np.testing.assert_array_equal(events[:b.n_events], want_ev, err_msg="call %d" % k)
            np.testing.assert_array_equal(calls, coracle.vote(want, 1), err_msg="call %d" % k)
    finally:
        ctx.close()
    dev = engine.require_cuda()
    table = engine.CountTable(seq[0][0].n_slots, dev)
    for k, (b, want, want_ev) in enumerate(seq):
        db = engine.upload(b, dev)
        if want is None:
            with pytest.raises(IndexError):
                engine.pileup(db, table=table)
            continue
        counts, events = engine.pileup(db, table=table)
        calls = engine.vote(counts, 1)
        torch.cuda.synchronize()
        np.testing.assert_array_equal(counts.cpu().numpy(), want, err_msg="pileup %d" % k)
        np.testing.assert_array_equal(events.cpu().numpy(), want_ev, err_msg="pileup %d" % k)
        np.testing.assert_array_equal(calls.cpu().numpy(), coracle.vote(want, 1), err_msg="pileup %d" % k)
