"""Base-quality, mapping-quality and flag filters (extension) on the CPU: the three decoders agree, the defaults
change nothing, the device correction K1q (run from its CUDA source in the emulator) equals the masking C oracle,
masks shard with their reads, and the CLI / REPORT expose the options."""
import os
import random

import numpy as np
import pytest

import emu_harness
from fuzz_cases import random_case
from kindel_b200 import bamio, cli, kindel, synth
from kindel_b200 import distributed as D
from oracle import qoracle

THRESHOLDS = (0, 1, 20, 41, 94)
ARRAYS = ("ref_start", "seq_off", "l_seq", "seq_len", "seq4", "complex_idx", "hard_idx", "contig_read_off",
          "contig_len", "cig_off", "cigar", "mask_read", "mask_off", "mask_qpos")


def with_fields(text, seed, qual_prob=0.85):
    """A fuzz case with random MAPQs, extra FLAG bits and Phred qualities (QUAL `*` for some records)."""
    rng = random.Random(seed * 7919 + 1)
    out = []
    for line in text.splitlines():
        if line.startswith("@"):
            out.append(line)
            continue
        f = line.split("\t")
        f[4] = str(rng.choice([0, 1, 5, 20, 30, 60, 255]))
        f[1] = str(int(f[1]) | rng.choice([0, 0, 0, 256, 1024, 2048, 512]))
        if f[9] != "*" and rng.random() < qual_prob:
            f[10] = "".join(chr(33 + rng.choice([0, 1, 2, 10, 19, 20, 21, 30, 40, 41, 93])) for _ in f[9])
        out.append("\t".join(f))
    return "\n".join(out) + "\n"


def sam_to_bam(text, path):
    """The same records through bamio.write_bam (binary BAM: MAPQ and QUAL bytes, 0xff for `*`)."""
    contigs, recs = [], []
    for line in text.splitlines():
        f = line.split("\t")
        if line.startswith("@SQ"):
            kv = dict(x.split(":", 1) for x in f[1:])
            contigs.append((kv["SN"], int(kv["LN"])))
            continue
        if line.startswith("@") or len(f) < 11:
            continue
        names = [c[0] for c in contigs]
        ref_id = names.index(f[2]) if f[2] in names else -1
        qual = None if f[10] == "*" else bytes(ord(c) - 33 for c in f[10])
        recs.append((ref_id, int(f[3]) - 1, int(f[1]), bamio.parse_cigar_text(f[5]), f[9], f[0], int(f[4]), qual))
    bamio.write_bam(path, contigs, recs)


def sam_quals(text):
    """Qualities of the reads read_sam keeps without filters, in its read order (0xff for QUAL `*`)."""
    groups = {}
    for line in text.splitlines():
        f = line.split("\t")
        if line.startswith("@") or len(f) < 11:
            continue
        g = groups.setdefault(f[2], [])
        if (int(f[1]) & 4) or len(f[9]) <= 1:
            continue
        g.append(b"\xff" * len(f[9]) if f[10] == "*" else bytes(ord(c) - 33 for c in f[10]))
    groups.pop("*", None)
    return np.frombuffer(b"".join(b"".join(g) for g in groups.values()), dtype=np.uint8)


def decode(fn, path, **kw):
    try:
        return fn(path, **kw)
    except (ValueError, KeyError) as e:
        return e


def same_arrays(a, b):
    for f in ARRAYS:
        x, y = getattr(a, f), getattr(b, f)
        assert (x is None) == (y is None), f
        if x is not None:
            assert np.array_equal(np.asarray(x), np.asarray(y)), f
    assert (a.n_events, a.reads_sorted, a.max_simple_len, a.reach_right, a.reach_left) == \
        (b.n_events, b.reads_sorted, b.max_simple_len, b.reach_right, b.reach_left)


@pytest.mark.parametrize("seed", range(0, 400, 5))
def test_decoders_agree(tmp_path, seed):
    text = with_fields(random_case(seed), seed)
    sam, bam = str(tmp_path / "c.sam"), str(tmp_path / "c.bam")
    with open(sam, "w") as fh:
        fh.write(text)
    sam_to_bam(text, bam)
    for thr in THRESHOLDS:
        for mq, ex in ((0, 0), (20, 0), (0, 0x400), (30, 0x900)):
            kw = dict(min_mapq=mq, exclude_flags=ex, min_base_quality=thr)
            py = decode(bamio.read_sam, sam, **kw)
            if isinstance(py, Exception):
                continue  # (an RNAME without @SQ line, a base BAM cannot hold: what the reference's path raises)
            cpp_sam = bamio.read_bam(sam, **kw)     # the C++ text parser takes these fields
            cpp_bam = bamio.read_bam(bam, **kw)
            same_arrays(cpp_sam, py)
            same_arrays(cpp_bam, py)
            if thr == 0:
                assert py.n_masked == 0


def test_defaults_are_identical(tmp_path):
    text = with_fields(random_case(11), 11)
    sam, bam = str(tmp_path / "c.sam"), str(tmp_path / "c.bam")
    with open(sam, "w") as fh:
        fh.write(text)
    sam_to_bam(text, bam)
    for path in (sam, bam):
        same_arrays(bamio.read_alignment(path), bamio.read_alignment(path, min_mapq=0, exclude_flags=0,
                                                                    min_base_quality=0))
        assert bamio.read_alignment(path, min_base_quality=0).n_masked == 0
    # a garbage QUAL changes nothing while the options are off, and is refused when the base filter reads it
    garbage = "\n".join(l if l.startswith("@") else "\t".join(l.split("\t")[:10] + ["\x7f!"]) for l in text.splitlines())
    g = str(tmp_path / "g.sam")
    with open(g, "w") as fh:
        fh.write(garbage + "\n")
    same_arrays(bamio.read_alignment(g), bamio.read_alignment(sam))
    with pytest.raises(ValueError):
        bamio.read_alignment(g, min_base_quality=20)
    # QUAL `*` (SAM) / 0xff (BAM) is never masked, at any threshold
    star = "\n".join(l if l.startswith("@") else "\t".join(l.split("\t")[:10] + ["*"]) for l in text.splitlines())
    s2, b2 = str(tmp_path / "s.sam"), str(tmp_path / "s.bam")
    with open(s2, "w") as fh:
        fh.write(star + "\n")
    sam_to_bam(star, b2)
    for path in (s2, b2):
        assert bamio.read_alignment(path, min_base_quality=255).n_masked == 0


def test_masked_exotic_base_is_simple_and_does_not_raise(tmp_path):
    head = "@SQ\tSN:c0\tLN:20\n"
    for qual, thr, raises in (("II#II", 20, False), ("IIIII", 20, True), ("II#II", 0, True)):
        p = str(tmp_path / "r.sam")
        with open(p, "w") as fh:
            fh.write(head + "r0\t0\tc0\t3\t60\t5M\t*\t0\t0\tACRGT\t%s\n" % qual)
        batch = bamio.read_alignment(p, min_base_quality=thr)
        qual_bytes = np.frombuffer(bytes(ord(c) - 33 for c in qual), dtype=np.uint8)
        if raises:
            with pytest.raises(KeyError) as e:
                qoracle.pileup(bamio.read_alignment(p), qual_bytes, thr)
            assert e.value.args == ("R",)
            with pytest.raises(KeyError) as e:
                emu_harness.pileup_pipeline(batch)
            assert e.value.args == ("R",)
        else:
            assert batch.n_masked == 1 and not batch.n_complex  # masked R reads as N: a simple read
            want, _ = qoracle.pileup(bamio.read_alignment(p), qual_bytes, thr)
            got, _ = emu_harness.pileup_pipeline(batch)
            assert np.array_equal(emu_harness.unmask(batch, got), want)
            assert want[4].sum() == 0 and want[0:4].sum() == 4


def _emu_vs_oracle(text, thr):
    import tempfile

    with tempfile.NamedTemporaryFile("w", suffix=".sam", delete=False) as fh:
        fh.write(text)
        path = fh.name
    try:
        try:
            plain = bamio.read_sam(path)
            masked = bamio.read_sam(path, min_base_quality=thr)
        except (ValueError, KeyError):
            return None
    finally:
        os.unlink(path)
    qual = sam_quals(text)
    try:
        want = qoracle.pileup(plain, qual, thr)
    except (IndexError, KeyError) as e:
        want = e
    try:
        counts, events = emu_harness.pileup_pipeline(masked)
        got = (emu_harness.unmask(masked, counts), events)
    except (IndexError, KeyError) as e:
        got = e
    if isinstance(want, Exception) or isinstance(got, Exception):
        assert type(want) is type(got)
        if isinstance(want, KeyError):
            assert want.args == got.args
    else:
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    return masked.n_masked


@pytest.mark.skipif(not emu_harness.available(), reason="needs g++ and the CUDA headers")
@pytest.mark.parametrize("schedule", ["forward", "reverse", "random"])
def test_k1q_emulated_equals_masking_oracle(schedule):
    emu_harness.set_schedule(schedule, 5)
    seeds = range(400) if schedule == "forward" else range(0, 400, 4)
    total = 0
    try:
        for seed in seeds:
            total += _emu_vs_oracle(with_fields(random_case(seed), seed), THRESHOLDS[seed % 4 + 1]) or 0
    finally:
        emu_harness.set_schedule("forward")
    assert total > 0


@pytest.mark.skipif(not emu_harness.available(), reason="needs g++ and the CUDA headers")
def test_k1q_emulated_on_synthetic_reads(monkeypatch):
    """Tile-eligible complex reads, hard reads (POS 0 wrap, overhanging right clips) and the depth split."""
    for seed, batch in ((1, synth.complex_reads(1, 4000, 60)), (2, synth.mixed_reads(3, [20000], 30, 0.1))):
        masked, qual = synth.with_qualities(batch, seed)
        assert masked.n_masked > 0 and masked.n_hard > 0 or seed == 2
        want = qoracle.pileup(batch, qual, 20)
        for split in (1, 3):
            monkeypatch.setenv("KDL_SPLIT", str(split))
            counts, events = emu_harness.pileup_pipeline(masked)
            assert np.array_equal(emu_harness.unmask(masked, counts), want[0])
            assert np.array_equal(events, want[1])


def test_masks_shard_with_their_reads(tmp_path):
    full, _ = synth.with_qualities(synth.complex_reads(5, 6000, 120), 9)
    counts_full = full.mask_counts()
    start = np.zeros(full.n_reads, dtype=np.int64)
    start[full.mask_read.astype(np.int64)] = full.mask_off[:-1]
    seen = 0
    for rank in range(3):
        idx = D.shard_indices(full, rank, 3, "reads")
        shard = D.shard_batch(full, rank, 3)
        c = shard.mask_counts()
        assert np.array_equal(c, counts_full[idx])
        s = np.zeros(shard.n_reads, dtype=np.int64)
        if shard.n_masked:
            s[shard.mask_read.astype(np.int64)] = shard.mask_off[:-1]
        for j, r in enumerate(idx.tolist()):
            assert np.array_equal(shard.mask_qpos[s[j]:s[j] + c[j]], full.mask_qpos[start[r]:start[r] + counts_full[r]])
        seen += shard.n_masked
        bamio.save_batch(str(tmp_path / ("s%d" % rank)), shard)
        same_arrays(bamio.load_batch(str(tmp_path / ("s%d" % rank))), shard)
    assert seen == full.n_masked
    # an unmasked batch saved over a masked one's directory loads unmasked
    plain = synth.complex_reads(5, 6000, 20)
    bamio.save_batch(str(tmp_path / "s0"), plain)
    assert bamio.load_batch(str(tmp_path / "s0")).n_masked == 0
    # merging keeps every read's mask
    merged = bamio.merge_batches([full, plain])
    assert merged.n_masked == full.n_masked


def test_cli_exposes_the_filters():
    p = cli.build_parser()
    for cmd in ("consensus", "weights", "features", "variants"):
        a = p.parse_args([cmd, "x.bam", "--min-base-quality", "20", "--min-mapq", "5", "--exclude-flags", "0x904"])
        assert (a.min_base_quality, a.min_mapq, a.exclude_flags) == (20, 5, 0x904)
        a = p.parse_args([cmd, "x.bam", "--exclude-flags", "1024"])
        assert (a.min_base_quality, a.min_mapq, a.exclude_flags) == (0, 0, 1024)


def test_report_lines():
    args = ("ref", kindel.DepthRange(1, 5), [None, "N"], None, "x.bam", False, 1, 7, 0.1, False, False)
    plain = kindel.build_report(*args)
    assert kindel.build_report(*args, filters=(0, 0, 0)) == plain
    assert "min_base_quality" not in plain
    lines = kindel.build_report(*args, filters=(20, 0, 0x900)).splitlines()
    at = lines.index("- uppercase: False")
    assert lines[at + 1:at + 4] == ["- min_base_quality: 20", "- min_mapq: 0", "- exclude_flags: 0x900"]
    assert [l for l in lines if l not in lines[at + 1:at + 4]] == plain.splitlines()


def test_new_symbols_are_exported():
    from kindel_b200 import _ffi

    lib = _ffi.load()
    for name in ("kdl_unmask", "kdl_ctx_consensus_masked", "kdl_bam_set_filter", "kdl_bam_fill_mask"):
        assert name in _ffi.EXPORTED_SYMBOLS and getattr(lib, name)
