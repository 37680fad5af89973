"""Bloom structures on the sharded path against the reference's goldens.

`count --bc`: every shard loads the whole counter and the sender drops a k-mer that fails it before routing it, so the
rank-ordered concatenation of the shard dumps is the reference's database byte for byte (golden_bc.json).  `count
--bf-size`: every shard keeps a filter for its share of the k-mers and applies it on the owner, after the exchange, where
every occurrence of a key arrives; the result is held to the contract of the single-GPU prefilter (count in {occ - 1, occ},
every k-mer seen twice present, false positives as many as the reference lets through).  `bc` across ranks: counters of
parts of the text folded into one (jfgpu_bloom_words / _fold / _dump_range) are the reference's file byte for byte.

Most tests run every shard's engine on one device, the data path of the multi-GPU commands without NCCL; the torchrun
tests need as many GPUs as ranks.

Cases left out: a shard never doubles, so no case whose reference table doubled -- bc_k40 (its count at -s 100k ends at
2^20 slots), bf_fp10_grow and bf_k40 (-s 100k, end at 2^19) -- and bf_q, whose -Q count_multi does not take.
"""
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest

import jfutil
from cases import BC_CASES, BF_CASES

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN_BC = json.load(open(os.path.join(HERE, "golden", "golden_bc.json")))
GOLDEN_BF = json.load(open(os.path.join(HERE, "golden", "golden_bf.json")))
BC_SHARD_CASES = ["bc_k21C", "bc_k63C", "bc_tiny"]
BF_SHARD_CASES = ["bf_fq", "bf_k63", "bf_small", "bf_twice"]
UINT64_MAX = (1 << 64) - 1


def _ngpu():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


def _size(v):
    return int(v[:-1]) * {"k": 10**3, "M": 10**6, "G": 10**9}[v[-1]] if v[-1] in "kMG" else int(v)


def _opts(args):
    """-> (global size, engine keyword arguments, dump keyword arguments) of a case's count switches"""
    rest = [a for a in args if a != "-C"]
    o = dict(zip(rest[0::2], rest[1::2]))
    eng = {"k": int(o["-m"]), "canonical": "-C" in args}
    if "--bf-size" in o:
        eng["bf_size"] = _size(o["--bf-size"])
        eng["bf_fp"] = float(o.get("--bf-fp", 0.01))
    dump = {"lower": int(o.get("-L", 0)), "upper": int(o.get("-U", UINT64_MAX)), "out_counter_len": int(o.get("--out-counter-len", 4))}
    return _size(o["-s"]), eng, dump


class Shards(object):
    """`world` engines of one global table on the current device.  File i is routed by shard i mod world
    (jfgpu_extract_route), its keys handed to their owners (jfgpu_insert_keys).  staged: the owners fill their tables
    region by region (part_min_mb = 1), else they insert directly."""

    def __init__(self, size, world, staged, bc=None, cap=1 << 20, **eng):
        import torch
        from jellyfish_b200 import HashCounter
        self.world = world
        # (every shard's record pool on the same device: 256 MB each rather than a share of the free memory)
        part = {"part_min_mb": 1, "pool_bytes": 256 << 20} if staged else {"no_partition": True}
        self.hcs = [HashCounter(size, 7, shard_index=r, n_shards=world, allow_regrow=False, max_batch_bytes=1 << 20, **dict(eng, **part))
                    for r in range(world)]
        if bc:
            for hc in self.hcs:
                hc.load_bloom_counter(bc)
        kw = self.hcs[0].key_words
        self.cap, self.kw = cap, kw
        self.keys = torch.zeros((world, cap * kw), dtype=torch.int64, device="cuda")
        self.counts = torch.zeros(world, dtype=torch.int64, device="cuda")
        self.n_files = 0

    def staged(self):
        return all(hc.info()["part_regions"] > 0 for hc in self.hcs)

    def add(self, data, chunk=200000):
        import torch
        router = self.hcs[self.n_files % self.world]
        self.n_files += 1
        a = 0
        while True:
            b = min(a + chunk, len(data))
            while b < len(data) and b - a > 1 and data[b - 1] == 13:      # (no piece but the last ends on '\r')
                b -= 1
            # every piece in a buffer of its own: device text starts 16-byte aligned, and a call reads nothing outside it
            buf = torch.zeros(b - a + 256, dtype=torch.uint8, device="cuda")
            if b > a:
                buf[:b - a] = torch.frombuffer(bytearray(data[a:b]), dtype=torch.uint8).cuda()
            self.counts.zero_()
            torch.cuda.synchronize()
            router.extract_route(buf.data_ptr(), b - a, self.keys.data_ptr(), self.cap, self.counts.data_ptr(),
                                 begin=a == 0, end=b >= len(data))
            c = self.counts.tolist()
            assert max(c) <= self.cap
            for d in range(self.world):
                self.hcs[d].insert_keys(self.keys[d].data_ptr(), c[d])
            a = b
            if a >= len(data):
                break

    def dump(self, out, **dump):
        from jellyfish_b200.distributed import concat_shards
        stats = []
        for r, hc in enumerate(self.hcs):
            stats.append(hc.done())
            hc.dump("%s.%d" % (out, r), **dump)
        return stats, jfutil.split_db(concat_shards(out, self.world, out + ".jf"))

    def close(self):
        for hc in self.hcs:
            hc.close()


def _bc_file(workdir, inputs, name):
    """the counter of a BC case written by the single-GPU `bc` (tests/test_gpu_parity.py holds it to the golden)"""
    bargs, bins, _, _ = BC_CASES[name]
    path = os.path.join(workdir, "shb_%s.bc" % name)
    if not os.path.exists(path):
        jfutil.run([jfutil.OUR_JF, "bc"] + bargs + ["-o", path] + [inputs[i] for i in bins])
    return path


@pytest.mark.parametrize("staged", [False, True])
@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("name", BC_SHARD_CASES)
def test_sharded_count_through_bloom_counter_matches_golden(name, world, staged, built, workdir, inputs):
    _, _, cargs, cins = BC_CASES[name]
    g = GOLDEN_BC[name]
    size, eng, dump = _opts(cargs)
    bc = _bc_file(workdir, inputs, name)
    sh = Shards(size, world, staged, bc=bc, **eng)
    try:
        if staged and not sh.staged():
            pytest.skip("a shard table of %d slots is under 1 MB: no region staging" % (size // world))
        for f in cins:
            sh.add(open(inputs[f], "rb").read())
        stats, (h, b) = sh.dump(os.path.join(workdir, "shb_bc_%s_%d_%d" % (name, world, staged)), **dump)
    finally:
        sh.close()
    assert jfutil.semantic(h) == g["header"]
    assert len(b) == g["body_len"] and jfutil.md5(b) == g["body_md5"]


def _unfiltered(name):
    """a BF case's switches without the filter, and its inputs"""
    args, ins = BF_CASES[name]
    plain = list(args)
    for sw in ("--bf-size", "--bf-fp"):
        if sw in plain:
            i = plain.index(sw)
            del plain[i:i + 2]
    return plain, ins


def check_prefilter_contract(name, h, b, workdir, inputs):
    """The contract of the single-GPU prefilter (tests/test_gpu_parity.py::test_bloom_prefilter_against_reference_golden)."""
    g = GOLDEN_BF[name]
    assert jfutil.semantic(h) == g["header"]
    plain, ins = _unfiltered(name)
    ref = os.path.join(workdir, "shb_occ_%s.jf" % name)
    if not os.path.exists(ref):
        jfutil.run([jfutil.ORACLE_C, "count"] + plain + ["-o", ref] + [inputs[i] for i in ins])
    hr, br = jfutil.split_db(ref)
    occ = dict(jfutil.records(hr, br))
    got = dict(jfutil.records(h, b))
    assert set(got) <= set(occ)
    cap = (1 << (8 * h["counter_len"])) - 1
    bad = [k for k, v in got.items() if v not in (min(occ[k], cap), min(occ[k] - 1, cap))]
    assert not bad, "counts outside {occ-1, occ}: %d" % len(bad)
    missing = [k for k in occ if k not in got and occ[k] > 1]
    assert not missing, "k-mers seen more than once must be present: %d missing" % len(missing)
    singles = [k for k in occ if occ[k] == 1]
    passed = sum(1 for k in singles if k in got)
    rec = (h["key_len"] + 7) // 8 + h["counter_len"]
    ref_passed = g["body_len"] // rec - (len(occ) - len(singles))
    assert 0 <= ref_passed <= len(singles)
    assert abs(passed - ref_passed) <= 50 + 0.05 * ref_passed + 4 * ref_passed ** 0.5, \
        "false positives: %d of %d singletons, reference %d" % (passed, len(singles), ref_passed)
    return occ, got


@pytest.mark.parametrize("staged", [False, True])
@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("name", BF_SHARD_CASES)
def test_sharded_prefilter_on_the_owner_meets_the_contract(name, world, staged, built, workdir, inputs):
    args, ins = BF_CASES[name]
    size, eng, dump = _opts(args)
    sh = Shards(size, world, staged, **eng)
    try:
        if staged and not sh.staged():
            pytest.skip("a shard table of %d slots is under 1 MB: no region staging" % (size // world))
        for f in ins:
            sh.add(open(inputs[f], "rb").read())
        stats, (h, b) = sh.dump(os.path.join(workdir, "shb_bf_%s_%d_%d" % (name, world, staged)), **dump)
        m_shard = sh.hcs[0].bloom_info()["m"]
    finally:
        sh.close()
    # a shard's filter is sized for its share of the expected k-mers, with the bits per k-mer of the single filter
    assert m_shard == (eng["bf_size"] + world - 1) // world * round(-math.log(eng["bf_fp"]) / math.log(2) ** 2)
    # (bf_twice: plain.fa is routed by shard 0 and again by shard 1; a filter on the sender would drop a first occurrence
    # on each side, occ - 2, and lose the k-mers seen once in each copy -- the contract's "seen twice, present")
    check_prefilter_contract(name, h, b, workdir, inputs)


def test_sharded_prefilter_draws_its_matrices_on_a_rank_that_routed_nothing(built, workdir, inputs):
    """An owner that receives keys before it has routed any text draws the filter's matrices itself: the same ones as
    every other shard (and the single filter)."""
    from jellyfish_b200 import HashCounter
    import torch
    a = HashCounter(1 << 20, 7, k=21, canonical=True, shard_index=0, n_shards=2, allow_regrow=False, bf_size=100000)
    b = HashCounter(1 << 20, 7, k=21, canonical=True, shard_index=1, n_shards=2, allow_regrow=False, bf_size=100000)
    one = HashCounter(1 << 20, 7, k=21, canonical=True, bf_size=100000)
    try:
        keys = torch.zeros(16, dtype=torch.int64, device="cuda")
        b.insert_keys(keys.data_ptr(), 1)
        ib, ia, i1 = b.bloom_info(), a.bloom_info(), one.bloom_info()
        assert ib["matrix1"] == ia["matrix1"] == i1["matrix1"] and ib["matrix2"] == ia["matrix2"] == i1["matrix2"]
        assert ib["m"] == ia["m"] == i1["m"] // 2
    finally:
        a.close(); b.close(); one.close()


def test_record_exchange_declines_bloom_engines(built):
    """jfgpu_shard_setup declines an engine with a Bloom structure, and one attached after setup makes
    jfgpu_shard_extract fail rather than be ignored."""
    from jellyfish_b200 import HashCounter, JellyfishError
    from jellyfish_b200 import _lib as L
    import torch
    big = dict(k=21, canonical=True, shard_index=0, n_shards=2, allow_regrow=False, part_min_mb=1)
    with HashCounter(1 << 22, 7, bf_size=1 << 20, **big) as hc:
        assert not hc.shard_setup(0, 0, 0, 0, 0, 0)
    with HashCounter(1 << 22, 7, **big) as hc:
        if not hc.shard_setup(0, 0, 0, 0, 0, 0):
            pytest.skip("geometry not covered by the record exchange")
        n_sm = torch.cuda.get_device_properties(0).multi_processor_count
        arena = 2 * n_sm * 1024 + 64
        send = torch.empty(2 * 2 * arena * 8192, dtype=torch.uint8, device="cuda")
        sdir = torch.empty(2 * 2 * arena * 8, dtype=torch.uint8, device="cuda")
        recv = torch.empty(2 * arena * 8192, dtype=torch.uint8, device="cuda")
        rdir = torch.empty(2 * arena * 8, dtype=torch.uint8, device="cuda")
        assert hc.shard_setup(send.data_ptr(), sdir.data_ptr(), arena, recv.data_ptr(), rdir.data_ptr(), arena)
        ctr = _bc_counter_bytes()
        hc._check(hc._lib.jfgpu_bloom_load(hc._h, ctr["m"], 3, ctr["m1"], ctr["m2"], ctr["body"], len(ctr["body"])))
        text = torch.zeros(4096, dtype=torch.uint8, device="cuda")
        with pytest.raises(JellyfishError) as ei:
            hc.shard_extract(text.data_ptr(), 100, 0)
        assert ei.value.code == L.ERR_STATE


def _bc_counter_bytes():
    import ctypes as C
    m = 1000
    return {"m": m, "m1": (C.c_uint64 * 42)(*range(1, 43)), "m2": (C.c_uint64 * 42)(*range(2, 44)), "body": bytes((m + 4) // 5)}


# -- bc across ranks ----------------------------------------------------------------------------------------------------------

def _words_tensor(ptr, n):
    import torch
    from jellyfish_b200.distributed import _DeviceWords
    return torch.as_tensor(_DeviceWords(ptr, n), device="cuda")


def _model_fold(a, b):
    a = a.astype(np.uint32)
    b = b.astype(np.uint32)
    return a | b | ((a & b & np.uint32(0x55555555)) << np.uint32(1))


def _model_pack(words, m):
    """file body of a counter in the two-bit form: five base-3 digits (hit + hit again) per byte"""
    pos = np.arange(m, dtype=np.uint64)
    f = (words[(pos >> np.uint64(4)).astype(np.int64)] >> ((pos & np.uint64(15)) * np.uint64(2)).astype(np.uint32)) & np.uint32(3)
    d = (f & 1) + (f >> 1)
    nb = (m + 4) // 5
    d = np.concatenate([d, np.zeros(5 * nb - m, d.dtype)]).reshape(nb, 5).astype(np.uint32)
    return (d * np.array([1, 3, 9, 27, 81], np.uint32)).sum(axis=1).astype(np.uint8).tobytes()


def _random_states(rng, n_words, m):
    """words whose positions < m hold a valid state (00, 01 or 11) and the rest 0"""
    st = rng.choice(np.array([0, 1, 3], np.uint32), size=n_words * 16)
    st[m:] = 0
    return (st.reshape(n_words, 16) << (np.arange(16, dtype=np.uint32) * 2)).sum(axis=1, dtype=np.uint64).astype(np.uint32)


def test_fold_kernel_against_model(built):
    import torch
    from jellyfish_b200 import BloomCounter
    rng = np.random.default_rng(5)
    with BloomCounter(1001, 0.001, k=17) as x, BloomCounter(1001, 0.001, k=17) as y:
        m = x.info()["m"]
        assert m % 16 and m % 5                      # a partial last word and a partial last byte
        px, n = x.words()
        py, ny = y.words()
        assert n == ny == (m + 15) // 16
        wx, wy = _random_states(rng, n, m), _random_states(rng, n, m)
        tx, ty = _words_tensor(px, n), _words_tensor(py, n)
        tx.copy_(torch.from_numpy(wx.view(np.int32)))
        ty.copy_(torch.from_numpy(wy.view(np.int32)))
        torch.cuda.synchronize()
        model = wx.copy()
        # ranges on and off the 5-word grid, to the last word, and empty
        for first, cnt in ((0, 5), (3, 17), (7, n - 7 - 2), (n - 4, 4), (12, 0), (20, 1)):
            x.fold(py + 4 * first, first, cnt)
            model[first:first + cnt] = _model_fold(model[first:first + cnt], wy[first:first + cnt])
        torch.cuda.synchronize()
        got = tx.cpu().numpy().view(np.uint32)
        assert np.array_equal(got, model)
        body = _model_pack(model, m)
        out = []
        x.dump_range(0, len(body), out.append)
        assert b"".join(out) == body
        for first, cnt in ((16, 32), (len(body) // 16 * 16, len(body) - len(body) // 16 * 16), (48, 0)):
            out = []
            x.dump_range(first, cnt, out.append)
            assert b"".join(out) == body[first:first + cnt]
        from jellyfish_b200 import JellyfishError
        with pytest.raises(JellyfishError):
            x.dump_range(8, 16, out.append)           # not on the 16-byte grid
        with pytest.raises(JellyfishError):
            x.fold(py, n - 2, 3)                      # past the last word


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("name", sorted(BC_CASES))
def test_bloom_counters_of_parts_folded_match_golden(name, world, built, workdir, inputs):
    """G counters on one device, each of the files files[r::G], folded slice by slice into the owner of the slice and
    dumped there: the concatenation is the reference's file, and count --bc through it gives the reference's database."""
    import torch
    from jellyfish_b200 import BloomCounter
    from jellyfish_b200.distributed import bloom_byte_range, bloom_slices, concat_bloom_slices
    bargs, bins, cargs, cins = BC_CASES[name]
    g = GOLDEN_BC[name]
    rest = [a for a in bargs if a != "-C"]
    o = dict(zip(rest[0::2], rest[1::2]))
    files = [inputs[i] for i in bins]
    share = [files[r::world] for r in range(world)]
    if name == "bc_k21C" and world == 4:
        assert share[0] == share[2] and not share[3]     # the same file on two ranks, and a rank with no text
    bcs = [BloomCounter(_size(o["-s"]), float(o.get("-f", 0.001)), k=int(o["-m"]), canonical="-C" in bargs) for _ in range(world)]
    try:
        for r in range(world):
            bcs[r].add_files(share[r])
        words = [bc.words() for bc in bcs]
        n = words[0][1]
        nb = bcs[0].info()["nb_bytes"]
        out = os.path.join(workdir, "shb_fold_%s_%d.bc" % (name, world))
        for r, (b, e) in enumerate(bloom_slices(n, world)):
            for s in range(world):
                if s != r and e > b:
                    bcs[r].fold(words[s][0] + 4 * b, b, e - b)
            torch.cuda.synchronize()
            fb, fe = bloom_byte_range(b, e, n, nb)
            with open("%s.%d" % (out, r), "wb") as f:
                bcs[r].dump_range(fb, fe - fb, f.write)
        concat_bloom_slices(out, world, bcs[0].header())
    finally:
        for bc in bcs:
            bc.close()
    hb, bb = jfutil.split_db(out)
    assert {k: hb.get(k) for k in g["bc_header"]} == g["bc_header"]
    assert len(bb) == g["bc_len"] and jfutil.md5(bb) == g["bc_md5"]
    db = out + ".jf"
    jfutil.run([jfutil.OUR_JF, "count"] + cargs + ["--bc", out, "-o", db] + [inputs[i] for i in cins])
    h, b = jfutil.split_db(db)
    assert jfutil.semantic(h) == g["header"]
    assert jfutil.md5(b) == g["body_md5"]


# -- the commands under torchrun --------------------------------------------------------------------------------------------

def _torchrun(world, module, args, port):
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
                        "--master-addr", "127.0.0.1", "--master-port", str(port), "-m", module] + args,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600, cwd=jfutil.ROOT,
                       env=dict(os.environ, SOURCE_DATE_EPOCH="0"))
    assert r.returncode == 0, r.stdout.decode()[-3000:]


@pytest.mark.skipif(_ngpu() < 2, reason="needs at least 2 GPUs")
@pytest.mark.parametrize("world", [2, 4, 8])
def test_count_multi_and_bc_multi_under_torchrun(world, built, workdir, inputs):
    if _ngpu() < world:
        pytest.skip("needs %d GPUs" % world)
    bargs, bins, cargs, cins = BC_CASES["bc_k21C"]
    g = GOLDEN_BC["bc_k21C"]
    bc = os.path.join(workdir, "shb_multi_%d.bc" % world)
    _torchrun(world, "jellyfish_b200.bc_multi", bargs + ["-o", bc] + [inputs[i] for i in bins], 29661)
    hb, bb = jfutil.split_db(bc)
    assert {k: hb.get(k) for k in g["bc_header"]} == g["bc_header"]
    assert len(bb) == g["bc_len"] and jfutil.md5(bb) == g["bc_md5"]
    db = os.path.join(workdir, "shb_multi_bc_%d.jf" % world)
    _torchrun(world, "jellyfish_b200.count_multi", cargs + ["--bc", bc, "-o", db] + [inputs[i] for i in cins], 29662)
    h, b = jfutil.split_db(db)
    assert jfutil.semantic(h) == g["header"] and jfutil.md5(b) == g["body_md5"]
    args, ins = BF_CASES["bf_twice"]
    db = os.path.join(workdir, "shb_multi_bf_%d.jf" % world)
    _torchrun(world, "jellyfish_b200.count_multi", args + ["-o", db] + [inputs[i] for i in ins], 29663)
    h, b = jfutil.split_db(db)
    check_prefilter_contract("bf_twice", h, b, workdir, inputs)
