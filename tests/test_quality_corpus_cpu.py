"""The aimed -Q texts of tests/quality_corpus.py, without a GPU: every cell lands where the generator claims, relative to
the batch end E, the last window's start h and the last tile's start, for every (TILE, last tile) that
tests/test_gpu_quality_seams.py uses; and the text model's -Q symbols on those texts are pinned to the C restatement
(oracle/jf_oracle.c), as tests/test_text_model_cpu.py does for its inputs."""
import os

import numpy as np
import pytest

import jfutil
import quality_corpus as qc
import seam_corpus as sc
import text_model as tm

Q = ord("5")
GEOMETRIES = [(tile, r) for tile in sc.TILES for r in (16, 96, 256, tile - 16, tile)]


def _batch(tile, r):
    return (1 if r < tile - 1024 else 2) * tile + r


@pytest.mark.parametrize("tile,r", GEOMETRIES)
@pytest.mark.parametrize("k", [21, 65])
def test_cells_land_where_claimed(k, tile, r):
    batch = _batch(tile, r)
    assert batch % 16 == 0 and qc.last_tile(batch, tile) == r and batch > tile
    (text, placed), = qc.cell_texts(batch, tile, k, qc.aimed_cells(k, Q))
    assert len(placed) == len(qc.aimed_cells(k, Q))
    rebuilt = 0
    for j, p in enumerate(placed):
        E, h, e = p["E"], p["h"], len(p["eol"])
        assert E == (j + 1) * batch and h == E - r - qc.HALO
        # S1: a sequence line (behind its header) that holds h, its '\n' a bytes into the window
        assert text[p["s1"] - 1] == 10 and text[p["s1"] - 1 - len(b"@p%d" % j) - (e - 1)] == ord("@")
        assert p["s1"] <= h <= p["nl1"] == h + p["a"] and text[p["nl1"]] == 10
        assert all(c in b"ACGT" for c in text[p["s1"]:p["nl1"] - (e - 1)]) and (e == 1 or text[p["nl1"] - 1] == 13)
        assert text[p["nl1"] + 1] == ord("+")
        # H2 right in front of S2; S2 from E + s2_off on, at least k bases past E
        assert text[p["hs"]] == ord("@") and text[p["hs"] - 1] == 10 and text[p["s2"] - 1] == 10
        assert p["s2"] == E + p["s2_off"] and p["s2"] + p["l2"] >= E + k
        assert all(c in b"ACGT" for c in text[p["s2"]:p["s2"] + p["l2"]])
        assert text[p["s2"] + p["l2"]:p["s2"] + p["l2"] + e + 1] == p["eol"] + b"+"
        q = text[p["q2"]:p["q2"] + p["l2"]]
        lows = {E + o - p["s2"] for o in p["low"]}
        assert all(E - qc.prek(k) <= E + o < E for o in p["low"])
        assert all(q[i] == (p["lowq"] if i in lows else qc.GOOD) for i in range(p["l2"]))
        assert text[p["q2"] + p["l2"]:p["q2"] + p["l2"] + e] == p["eol"]
        # the header starts in the last tile exactly when the generator counts its reset outside the halo
        n, halo_reset = qc.window_symbols(p, Q)
        assert n >= max(0, E - p["s2"])
        rebuilt += qc.carry_is_rebuilt(p, k, Q, batch, tile)
        if qc.carry_is_rebuilt(p, k, Q, batch, tile) and p["hs"] < E:
            assert E - r <= p["hs"]
    # a short last tile leaves room for a header only at its very end; every other geometry rebuilds most carries
    assert rebuilt >= (5 if r == 16 else len(placed) // 2), rebuilt


def _oracle_counts(tmp, data, k, canonical, min_qual):
    path = os.path.join(tmp, "in.fq")
    with open(path, "wb") as f:
        f.write(data)
    out = os.path.join(tmp, "o.jf")
    cmd = [jfutil.ORACLE_C, "count", "-m", str(k), "-s", str(max(1024, 2 * len(data))), "-o", out, "--out-counter-len", "8"]
    jfutil.run(cmd + (["-C"] if canonical else []) + (["-Q", chr(min_qual)] if min_qual else []) + [path])
    h, b = jfutil.split_db(out)
    return tm.records_to_words(b, k, h["counter_len"])


@pytest.mark.parametrize("tile,r", [(sc.TILE_512, 96), (sc.TILE_512, 256), (sc.TILE_512, sc.TILE_512 - 16), (sc.TILE_1024, sc.TILE_1024)])
def test_model_matches_oracle_on_cells(tile, r, built, tmp_path):
    if not os.path.exists(jfutil.ORACLE_C):
        pytest.skip("oracle not built")
    k = 31
    batch = _batch(tile, r)
    cells = qc.aimed_cells(k, Q, full=False)
    for i, (text, _) in enumerate(qc.cell_texts(batch, tile, k, cells[::3], per_text=6)[:2]):
        for mq in (Q, 0):
            keys, cnt = _oracle_counts(str(tmp_path), text, k, i % 2 == 0, mq)
            mk, mc, _ = tm.counts(tm.symbols(text, mq), k, i % 2 == 0)
            assert np.array_equal(mk, keys) and np.array_equal(mc, cnt), "text %d -Q %r: model %d distinct, oracle %d" % (i, mq, len(mk), len(keys))


def test_filler_adds_resets_only():
    """The 512 MB case counts the model of the cell's two reads alone: the same k-mers as the whole text under -Q."""
    k = 21
    E = 3 * sc.TILE_1024 + 256 + (10 << 10) // sc.TILE_1024 * sc.TILE_1024
    text, body, place = qc.one_cell_text(E, sc.TILE_1024, k, qc.cell(-30, low=[-5, -17]), E + 30000)
    assert qc.last_tile(E, sc.TILE_1024) == 256 and qc.last_tile(512 << 20, sc.TILE_1024) == 256
    assert qc.carry_is_rebuilt(place, k, Q, E, sc.TILE_1024)
    assert text[place["s2"] - 1] == 10 and place["s2"] == E - 30
    whole = tm.counts(tm.symbols(text.tobytes(), Q), k, True)
    alone = tm.counts(tm.symbols(body, Q), k, True)
    assert np.array_equal(whole[0], alone[0]) and np.array_equal(whole[1], alone[1]) and whole[2] == alone[2] > 0
