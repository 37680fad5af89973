"""k-mers longer than 64 bases on the host, without a GPU: the hash matrices of 2k = 130..256 columns and the CPU readers
(dump, query, info, histo, stats, merge) of jellyfish-b200 on two small k = 100 databases written by the unmodified
reference (tests/golden/large_k_a.bin, large_k_b.bin), against the reference's own outputs
(tests/golden/golden_large_k.json, scripts/make_large_k_golden.py)."""
import ctypes as C
import json
import os

import pytest

import jfutil

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = json.load(open(os.path.join(HERE, "golden", "golden_large_k.json")))
HOST = GOLDEN["host"]
DB = {t: os.path.join(HERE, "golden", "large_k_%s.bin" % t) for t in ("a", "b")}


def ours(*args):
    return jfutil.run([jfutil.OUR_JF] + list(args), env={"CUDA_VISIBLE_DEVICES": ""}).stdout


@pytest.mark.parametrize("m", GOLDEN["matrices"], ids=lambda m: "r%d_c%d_skip%d" % (m["r"], m["c"], m["skip"]))
def test_reference_matrix_of_wide_keys(m, built):
    lib = C.CDLL(jfutil.LIB)
    cols = (C.c_uint64 * m["c"])()
    assert lib.jfgpu_reference_matrix(m["r"], m["c"], m["skip"], cols) == 0
    assert list(cols) == m["columns"]


def test_reference_matrix_rejects_more_than_256_columns(built):
    lib = C.CDLL(jfutil.LIB)
    cols = (C.c_uint64 * 257)()
    assert lib.jfgpu_reference_matrix(20, 257, 0, cols) != 0


@pytest.mark.parametrize("tag", ["a", "b"])
def test_dump(tag, built):
    g = HOST[tag]
    assert jfutil.md5(ours("dump", DB[tag])) == g["dump_md5"]
    assert jfutil.md5(ours("dump", "-c", "-t", DB[tag])) == g["dump_ct_md5"]
    assert jfutil.md5(ours("dump", "-c", "-L", "2", DB[tag])) == g["dump_L2_md5"]


@pytest.mark.parametrize("tag", ["a", "b"])
def test_query_mers_reverse_complements_and_wrong_lengths(tag, built):
    r = jfutil.run([jfutil.OUR_JF, "query", DB[tag]] + HOST["query_mers"], env={"CUDA_VISIBLE_DEVICES": ""})
    # the first 12 mers are valid 100-mers; the reference pads or reads past the 96-base and the N-bearing ones, which
    # jellyfish-b200 rejects (as for any k)
    assert r.stdout.decode().splitlines() == HOST[tag]["query"].splitlines()[:12]
    assert r.stderr.count(b"Invalid mer") == 2


@pytest.mark.parametrize("tag", ["a", "b"])
def test_query_sequence_on_the_cpu(tag, built, tmp_path):
    fa = tmp_path / "q.fa"
    fa.write_text(HOST["fasta_" + tag])
    assert jfutil.md5(ours("query", "-s", str(fa), DB[tag])) == HOST[tag]["query_s_md5"]


@pytest.mark.parametrize("tag", ["a", "b"])
def test_info_histo_stats(tag, built):
    g = HOST[tag]
    assert ours("info", DB[tag]).decode().split("\n")[1:] == g["info"].split("\n")[1:]
    assert ours("histo", DB[tag]).decode() == g["histo"]
    assert ours("stats", DB[tag]).decode() == g["stats"]


@pytest.mark.parametrize("op", ["sum", "min", "max"])
def test_merge(op, built, tmp_path):
    out = str(tmp_path / "m.jf")
    ours("merge", *({"sum": [], "min": ["--min"], "max": ["--max"]}[op]), "-o", out, DB["a"], DB["b"])
    h, b = jfutil.split_db(out)
    g = HOST["merge_" + op]
    assert jfutil.semantic(h) == g["header"]
    assert jfutil.md5(b) == g["body_md5"]


def test_merge_jaccard(built, tmp_path):
    out = str(tmp_path / "j.txt")
    ours("merge", "--jaccard", "-o", out, DB["a"], DB["b"])
    assert open(out).read() == HOST["merge_jaccard"]


def test_count_rejects_mers_longer_than_128_and_bloom_switches_beyond_64(built, tmp_path):
    fa = tmp_path / "x.fa"
    fa.write_text(">x\nACGT\n")
    for args in (["-m", "129", "-s", "1k"], ["-m", "100", "-s", "1k", "--bf-size", "1k"], ["-m", "65", "-s", "1k", "--bc", str(fa)]):
        r = jfutil.subprocess.run([jfutil.OUR_JF, "count"] + args + ["-o", str(tmp_path / "o.jf"), str(fa)],
                                  stdout=jfutil.subprocess.PIPE, stderr=jfutil.subprocess.PIPE)
        assert r.returncode != 0
        assert b"Error" in r.stderr
    r = jfutil.subprocess.run([jfutil.OUR_JF, "bc", "-m", "65", "-s", "1k", str(fa)], stdout=jfutil.subprocess.PIPE,
                              stderr=jfutil.subprocess.PIPE)
    assert r.returncode != 0 and b"1..64" in r.stderr
