"""CPU tests of `count_multi --disk`: the command line, the names of the pieces, and the end of a count on every rank --
each rank merges its own pieces, rank 0 concatenates -- against `merge` of whole databases."""
import os

import numpy as np
import pytest

import gen
import jfutil
from cases import DISK_PART_ARGS


def _parse(argv):
    from jellyfish_b200 import count_multi
    return count_multi.parse_args(argv)


def test_disk_with_if_is_refused(capsys):
    with pytest.raises(SystemExit) as ex:
        _parse(["-m", "21", "-s", "1M", "--disk", "--if", "a.fa", "b.fa"])
    assert ex.value.code == 1
    assert "--disk with --if" in capsys.readouterr().err
    a = _parse(["-m", "21", "-s", "1M", "--disk", "--no-merge", "--no-unlink", "b.fa"])
    assert a.disk and a.no_merge and a.no_unlink
    a = _parse(["-m", "21", "-s", "1M", "--if", "a.fa", "--no-merge", "b.fa"])
    assert not a.disk and a.no_merge


def test_piece_names():
    from jellyfish_b200.distributed import piece_path
    assert piece_path("out.jf", 0, 0) == "out.jf.0.0"
    assert piece_path("/d/x", 3, 12) == "/d/x.3.12"


def _info(header):
    m = header["matrix1"]
    return {"size": header["size"], "matrix_identity": m["identity"], "matrix_columns": m.get("columns"), "matrix_c": m["c"]}


def _recode(header, body, ocl, scale=1):
    """The records of a database with ocl count bytes, counts (times `scale`) clipped as a dump with --out-counter-len ocl
    clips them."""
    kb, cl = (header["key_len"] + 7) // 8, header["counter_len"]
    a = np.frombuffer(body, np.uint8).reshape(-1, kb + cl)
    counts = np.zeros(len(a), np.uint64)
    for j in range(cl):
        counts |= a[:, kb + j].astype(np.uint64) << np.uint64(8 * j)
    counts *= np.uint64(scale)
    counts = np.minimum(counts, np.uint64((1 << (8 * ocl)) - 1) if ocl < 8 else counts)
    out = np.zeros((len(a), kb + ocl), np.uint8)
    out[:, :kb] = a[:, :kb]
    for j in range(ocl):
        out[:, kb + j] = ((counts >> np.uint64(8 * j)) & np.uint64(255)).astype(np.uint8)
    return out


def _write_db(path, header, recs):
    from jellyfish_b200.engine import write_header
    with open(path, "wb") as f:
        write_header(f, header)
        f.write(recs.tobytes())


class _FakeEngine(object):
    """What DiskPieces needs of the engine: the shard as it stands (a piece) and its header."""

    def set_spill(self, fn):
        self.hook = fn

    def __init__(self, header):
        self.hdr = header
        self.table = None            # records of the shard as it stands

    def header(self, out_counter_len=4, cmdline=()):
        return dict(self.hdr, counter_len=out_counter_len, cmdline=list(cmdline))

    def dump(self, path, lower=0, upper=(1 << 64) - 1, out_counter_len=4, cmdline=()):
        kb = (self.hdr["key_len"] + 7) // 8
        recs = self.table
        if lower or upper != (1 << 64) - 1:
            c = np.zeros(len(recs), np.uint64)
            for j in range(out_counter_len):
                c |= recs[:, kb + j].astype(np.uint64) << np.uint64(8 * j)
            recs = recs[(c >= lower) & (c <= upper)]
        _write_db(path, self.header(out_counter_len, cmdline), recs)


@pytest.mark.parametrize("world", [1, 2, 4, 8])
def test_per_shard_merges_concatenated_equal_the_whole_merge(world, built, workdir, inputs):
    """Eight databases of one geometry (the pieces `merge` is checked on in test_host.py) stand for the pieces of a --disk
    count: each is cut by position range into the slices `world` shards would have written.  Every rank's pieces are merged
    by DiskPieces.write_output (the CLI's merge, -L/-U on the sums) and concat_shards joins the ranks: byte for byte the
    CLI's merge of the whole databases, for every counter length 1..8 and with -L/-U.  Three databases come twice, so that
    some sums are 2; with one count byte every count is 200, so that those sums clip (to 255, as the total would)."""
    from jellyfish_b200.distributed import DiskPieces, concat_shards
    d = os.path.join(workdir, "disk_multi_%d" % world)
    os.makedirs(d, exist_ok=True)
    parts = []
    for i, fa in enumerate(gen.disk_part_files(d, inputs["plain.fa"])):
        parts.append(os.path.join(d, "part%d.jf" % i))
        jfutil.run([jfutil.ORACLE_C, "count"] + DISK_PART_ARGS + ["-o", parts[-1], fa])
    dbs = [jfutil.split_db(p) for p in parts + parts[:3]]
    h0 = dbs[0][0]
    size, k = h0["size"], h0["key_len"] // 2
    kb = (h0["key_len"] + 7) // 8
    for ocl, lower, upper in [(4, 0, None), (1, 0, None), (2, 2, None), (3, 0, 1), (5, 2, 7), (6, 0, None), (7, 1, None), (8, 0, 5)]:
        whole, slices = [], [[] for _ in range(world)]
        for i, (h, b) in enumerate(dbs):
            recs = _recode(h, b, ocl, 200 if ocl == 1 else 1)
            hd = dict(h, counter_len=ocl)
            whole.append(os.path.join(d, "whole%d.jf" % i))
            _write_db(whole[-1], hd, recs)
            keys = np.zeros((len(recs), (2 * k + 63) // 64), np.uint64)
            for j in range(kb):
                keys[:, j // 8] |= recs[:, j].astype(np.uint64) << np.uint64(8 * (j % 8))
            owner = jfutil.positions(_info(h), keys, k) // np.uint64(size // world)
            for r in range(world):
                slices[r].append(recs[owner == r])
        want = os.path.join(d, "want.jf")
        switches = (["-L", str(lower)] if lower else []) + (["-U", str(upper)] if upper is not None else [])
        jfutil.run([jfutil.OUR_JF, "merge"] + switches + ["-o", want] + whole)
        out = os.path.join(d, "out.jf")
        for r in range(world):
            sc = DiskPieces(_FakeEngine(dict(h0, counter_len=ocl, canonical=True, val_len=7)), out, r, ocl)
            for recs in slices[r][:-1]:                 # the spills ...
                sc.hc.table = recs
                sc.hc.hook(sc.hc)
            sc.hc.table = slices[r][-1]                 # ... and the table at the end
            assert sc.pieces == ["%s.%d.%d" % (out, r, i) for i in range(len(dbs) - 1)]
            sc.write_output("%s.%d" % (out, r), lower, upper if upper is not None else (1 << 64) - 1, ["count_multi"])
            assert not any(os.path.exists(p) for p in sc.pieces)
        concat_shards(out, world, out)
        hw, bw = jfutil.split_db(want)
        ho, bo = jfutil.split_db(out)
        assert bo == bw, (ocl, lower, upper)
        assert len(bo) > 0, (ocl, lower, upper)
        if ocl == 1:
            assert 255 in set(bo[kb::kb + 1]) and 200 in set(bo[kb::kb + 1])
        # the merge's keys, and those of the count (the merge itself writes neither `canonical` nor `val_len`)
        assert {x: ho[x] for x in ("size", "key_len", "matrix1", "max_reprobe", "reprobes", "counter_len", "format")} == \
               {x: hw[x] for x in ("size", "key_len", "matrix1", "max_reprobe", "reprobes", "counter_len", "format")}
        assert ho["canonical"] is True and ho["val_len"] == 7


def test_rank_that_never_spilled_dumps_with_bounds_and_no_merge_keeps_pieces(tmp_path):
    """write_output: without a spill the shard goes straight to OUT.<rank> with -L/-U; merge=False leaves every piece
    (a rank that never spilled writes its table as its only piece) and no OUT.<rank>; unlink=False keeps merged pieces;
    discard_pieces (the fall-back of a failed cut check) deletes the pieces and restarts the numbering."""
    from jellyfish_b200.distributed import DiskPieces
    h = {"key_len": 8, "size": 16, "counter_len": 1, "format": "binary/sorted", "matrix1": {"r": 4, "c": 8, "identity": False,
         "columns": [1, 2, 4, 8, 3, 5, 6, 7]}, "max_reprobe": 3, "reprobes": [1, 1, 3, 6], "alignment": 8}
    recs = np.array([[1, 1], [2, 5], [3, 9]], np.uint8)
    recs = recs[np.argsort(jfutil.positions(_info(h), recs[:, :1].astype(np.uint64), 4), kind="stable")]     # (position order)
    out = str(tmp_path / "o.jf")

    def counter():
        sc = DiskPieces(_FakeEngine(h), out, 1, 1)
        sc.hc.table = recs
        return sc
    sc = counter()
    sc.write_output(out + ".1", lower=2, upper=8)
    assert jfutil.split_db(out + ".1")[1] == bytes([2, 5])
    assert sc.pieces == [] and not os.path.exists(out + ".1.0")
    os.unlink(out + ".1")
    sc = counter()
    sc.write_output(out + ".1", merge=False)
    assert sc.pieces == [out + ".1.0"] and os.path.exists(out + ".1.0") and not os.path.exists(out + ".1")
    sc.discard_pieces()
    assert sc.pieces == [] and not os.path.exists(out + ".1.0")
    sc.hc.hook(sc.hc)
    assert sc.pieces == [out + ".1.0"]
    sc.discard_pieces()
    sc.hc.hook(sc.hc)
    sc.write_output(out + ".1", unlink=False)
    assert sc.pieces == [out + ".1.0", out + ".1.1"] and all(os.path.exists(p) for p in sc.pieces)
    b = jfutil.split_db(out + ".1")[1]
    assert sorted(b[i:i + 2] for i in range(0, len(b), 2)) == [bytes([1, 2]), bytes([2, 10]), bytes([3, 18])]
