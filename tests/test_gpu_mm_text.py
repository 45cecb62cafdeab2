"""The MM text corpus (test_mm_text_cpu.py) through the product: for the default kernels, the fused (MKP_FUSED=1) and the tile
(MKP_TILE=1) kernels, every row against the independent model (mmmodel.py with callmodel.py) and the whole text against the
oracle, over all positions and with --cpg; then the default kernels under host ingest, a chunk size that splits the corpus and
two shards on one device; summary (its counts against the model's totals as well) and sample-probs; pileup-hemi on the duplex
variant. A read whose text the reference would
not use is in no count; a read it accepts gives the model's counts."""
import pytest

from conftest import run_oracle, run_product, same_text
from test_gpu_call_table import with_env
from test_hemi_cpu import hemi_oracle_exe  # noqa: F401 (fixture)
from test_mm_text_cpu import FLAG_SETS, build_corpus, check_rows, check_summary, write_corpus

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def corpus_files(tmp_path_factory):
    corpus = build_corpus()
    bam, fa, contig = write_corpus(corpus, tmp_path_factory.mktemp("mmtext"))
    return corpus, bam, fa, contig


@pytest.mark.parametrize("kernel", [None, "MKP_FUSED", "MKP_TILE"])
@pytest.mark.parametrize("name", ["all", "cpg", "cpg_force", "ignore_h", "combine_mods"])
def test_pileup_matches_model_and_oracle(name, kernel, corpus_files, native_lib, oracle_exe, tmp_path):
    corpus, bam, fa, contig = corpus_files
    flags = [fa if f == "FA" else f for f in dict(FLAG_SETS)[name]]
    exp = run_oracle(oracle_exe, flags, bam, str(tmp_path / "o.bed"))
    rc, got = with_env(kernel, lambda: run_product(flags, bam, str(tmp_path / "g.bed")))
    assert rc == 0
    n_rows, used, unused = check_rows(got, corpus, contig, flags)
    assert n_rows > 300 and used >= 200 and unused >= 100
    assert same_text(got, exp)


@pytest.mark.parametrize("variant", [["--host-ingest"], ["--gpu-chunk-bp", "50000"], ["--devices", "0,0"]], ids=lambda v: v[0][2:])
def test_pileup_invariant_under_ingest_chunks_and_shards(variant, corpus_files, native_lib, tmp_path):
    corpus, bam, fa, contig = corpus_files
    for flags in (["--no-filtering"], ["--no-filtering", "--cpg", "--ref", fa]):
        rc, got = run_product(flags + variant, bam, str(tmp_path / "g.bed"))
        assert rc == 0
        check_rows(got, corpus, contig, flags)


def test_reports_match_oracle(corpus_files, native_lib, oracle_exe, tmp_path):
    from test_gpu_summary import oracle, product
    corpus, bam, _, contig = corpus_files
    for cmd, args in (("summary", ["--tsv", "--no-sampling", "--no-filtering"]), ("summary", ["--tsv", "--no-sampling", "--no-filtering", "--ignore", "h"]),
                      ("sample-probs", ["--no-sampling", "-p", "0.1,0.5,0.9"])):
        exp = oracle(oracle_exe, cmd, args + [bam])
        assert exp.count("\n") > 3
        got = product(cmd, args + [bam], tmp_path)
        if cmd == "summary":                                     # reads used, reads and calls per base and code: the model's totals
            assert check_summary(got, corpus, "h" if "--ignore" in args else None) >= 200
        assert got == exp, (cmd, args)


def test_hemi_duplex_corpus_matches_oracle(native_lib, hemi_oracle_exe, tmp_path):
    from test_gpu_hemi import run_hemi, run_oracle_hemi
    bam, fa, _ = write_corpus(build_corpus(duplex=True), tmp_path, "duplex")
    for flags in (["--no-filtering"], ["--filter-threshold", "C:0.75"]):
        args = [bam, "-r", fa, "--cpg"] + flags
        exp = run_oracle_hemi(hemi_oracle_exe, args, str(tmp_path / "oh.bed"))
        assert exp.count("\n") > 200
        rc, got = run_hemi(args, str(tmp_path / "gh.bed"))
        assert rc == 0 and same_text(got, exp), flags
