"""The column corpus (test_pileup_columns_cpu.py) through the product: for the default per-stage kernels, the fused (MKP_FUSED=1)
and the tile (MKP_TILE=1) kernels, every flag set's text against the independent column model (pileupmodel.py) and against
the oracle, in all-positions mode and with focus bitmaps (--cpg, motif sets, --include-bed), with --combine-strands and
--combine-mods; then interval sizes and a chunk size whose word origins move through every bit, host ingest and two shards
on one device (against the model and the oracle); a --partition-tag run; the raw C ABI (upload / pileup_resident / fetch_rows),
whose row fields, primary base included, are checked against the model."""
import functools

import pytest

import pileupmodel as pm
from conftest import read_dir, run_oracle, run_product, same_text
from test_gpu_call_table import with_env
from test_pileup_columns_cpu import corpus_files, flags_of, model_text  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu

KERNEL_SETS = ["all_force", "thresholds", "edge", "ignore_h", "cpg", "motifs", "cgcg", "include", "cpg_include", "cpg_combine",
               "cgcg_combine", "combine_mods", "combine_mods_strands"]


@pytest.mark.parametrize("kernel", [None, "MKP_FUSED", "MKP_TILE"])
@pytest.mark.parametrize("name", KERNEL_SETS)
def test_pileup_columns_match_model_and_oracle(name, kernel, corpus_files, native_lib, oracle_exe, tmp_path):
    _, bam, fa, bed = corpus_files
    flags = flags_of(name, fa, bed)
    rc, got = with_env(kernel, lambda: run_product(flags, bam, str(tmp_path / "g.bed")))
    assert rc == 0
    assert same_text(got, model_text(bam, flags))
    assert same_text(got, run_oracle(oracle_exe, flags, bam, str(tmp_path / "o.bed")))


@pytest.mark.parametrize("name,extra", [("i25", []), ("i25", ["--gpu-chunk-bp", "990"]), ("cpg_i88", []), ("cpg_i88", ["--gpu-chunk-bp", "1000"]),
                                        ("cpg_combine_i25", ["--gpu-chunk-bp", "990"]), ("all", ["-i", "10000"]), ("all_force", ["--host-ingest"]),
                                        ("cpg", ["--host-ingest"]), ("all_force", ["--devices", "0,0"]), ("cpg_combine", ["--devices", "0,0"])],
                         ids=lambda v: "_".join(v) if isinstance(v, list) else v)
def test_pileup_columns_under_chunks_ingest_and_shards(name, extra, corpus_files, native_lib, oracle_exe, tmp_path):
    _, bam, fa, bed = corpus_files
    flags = flags_of(name, fa, bed)
    rc, got = run_product(flags + extra, bam, str(tmp_path / "g.bed"))
    assert rc == 0
    same = [f for f in flags + extra if f not in ("--gpu-chunk-bp", "990", "1000", "--host-ingest", "--devices", "0,0")]
    assert same_text(got, model_text(bam, same))
    assert same_text(got, run_oracle(oracle_exe, same, bam, str(tmp_path / "o.bed")))


def test_pileup_columns_partitions(corpus_files, native_lib, tmp_path):
    """--partition-tag HP: keys 1 and 2 and untagged reads share columns; each file against the model."""
    _, bam, _, _ = corpus_files
    flags = ["--no-filtering", "--force-allow-implicit", "--partition-tag", "HP"]
    rc, _ = run_product(flags, bam, str(tmp_path / "part"))
    assert rc == 0
    got, exp = read_dir(str(tmp_path / "part")), pm.partition_files(pm.load_bam(bam), flags)
    assert sorted(got) == sorted(exp) == ["1.bed", "2.bed", "ungrouped.bed"]
    for name in exp:
        assert same_text(got[name], exp[name]), name


@functools.lru_cache(maxsize=None)
def model_rows(bam):
    return pm.pileup(pm.load_bam(bam), ["--no-filtering", "--force-allow-implicit"])[0]


@pytest.mark.parametrize("contig", ["scn", "deep", "mot", "geo"])
def test_pileup_columns_raw_abi(contig, corpus_files, native_lib):
    """One contig through upload_chunk / pileup_resident / fetch_rows: every mkp_row field against the model's rows."""
    import modkit_b200
    corpus, bam, _, _ = corpus_files
    refs = [n for n in corpus.contigs]
    tid = refs.index(contig)
    b = modkit_b200.Bam(bam, threads=4)
    pk = b.pack(tid, 0, len(corpus.contigs[contig]))
    ctx = modkit_b200.Context(0)
    ctx.set_params(modkit_b200.make_params(force_allow_implicit=True))
    ctx.upload(pk)
    st = ctx.pileup_resident()
    rows = ctx.fetch_rows().copy()
    assert st.n_rows == len(rows) > 50
    got = sorted((int(r["pos"]), chr(r["strand"]), int(r["code"]), "ACGT"[r["primary_base"]], int(r["n_mod"]), int(r["n_canon"]),
                  int(r["n_other"]), int(r["n_delete"]), int(r["n_filtered"]), int(r["n_diff"]), int(r["n_nocall"])) for r in rows)
    out = model_rows(bam)
    exp = sorted((p, r.strand, ord(r.code) if isinstance(r.code, str) else 0x80000000 | r.code, r.primary, r.n_mod, r.n_canon,
                  r.n_other, r.n_delete, r.n_fail, r.n_diff, r.n_nocall) for c, p, r in out[None] if c == contig)
    assert got == exp, (len(got), len(exp), next((x, y) for x, y in zip(got, exp) if x != y) if got != exp else None)
