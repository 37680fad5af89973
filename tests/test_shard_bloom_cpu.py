"""CPU tests of the host logic of Bloom structures on several ranks: the slicing of a counter on the 5-word grid, the
reduce-scatter that folds every rank's counter into the slice it owns (gloo, worlds 2 and 3, pieces smaller than a slice,
the device fold replaced by numpy behind the `BloomBackend` seam), and the argument checks of count_multi."""
import os
import subprocess
import sys
import textwrap

import jfutil

WORKER = textwrap.dedent('''
    import os, sys
    import numpy as np, torch, torch.distributed as dist
    sys.path.insert(0, %(root)r)
    from jellyfish_b200.distributed import BloomBackend, bloom_byte_range, bloom_reduce_scatter

    M = %(m)d
    N_WORDS, N_BYTES = (M + 15) // 16, (M + 4) // 5

    def states(seed):
        st = np.random.default_rng(seed).choice(np.array([0, 1, 3], np.uint32), size=N_WORDS * 16)
        st[M:] = 0
        return (st.reshape(N_WORDS, 16) << (np.arange(16, dtype=np.uint32) * 2)).sum(axis=1, dtype=np.uint64).astype(np.uint32)

    def fold(a, b):
        return a | b | ((a & b & np.uint32(0x55555555)) << np.uint32(1))

    def pack(words, first_byte, n_bytes):
        out = bytearray()
        for j in range(first_byte, first_byte + n_bytes):
            v = 0
            for i in range(5):
                p = 5 * j + i
                if p < M:
                    f = (int(words[p >> 4]) >> (2 * (p & 15))) & 3
                    v += ((f & 1) + (f >> 1)) * 3 ** i
            out.append(v)
        return bytes(out)

    class NumpyBloomBackend(BloomBackend):
        n_words, n_bytes = N_WORDS, N_BYTES
        def __init__(self, words): self.w = torch.from_numpy(words.view(np.int32).copy()); self.folds = 0
        def words(self): return self.w
        def fold(self, words, first_word):
            mine = self.w[first_word:first_word + words.numel()]
            mine.copy_(torch.from_numpy(fold(mine.numpy().view(np.uint32), words.numpy().view(np.uint32)).view(np.int32)))
            self.folds += 1
        def dump_range(self, first_byte, n_bytes, sink): sink(pack(self.w.numpy().view(np.uint32), first_byte, n_bytes))

    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dist.init_process_group("gloo")
    be = NumpyBloomBackend(states(100 + rank))
    b, e = bloom_reduce_scatter(be, rank, world, piece_words=%(piece)d)
    want = states(100)
    for r in range(1, world):
        want = fold(want, states(100 + r))
    got = be.w.numpy().view(np.uint32)
    assert np.array_equal(got[b:e], want[b:e]), "rank %%d: slice differs" %% rank
    assert (e - b) > %(piece)d, "pieces must be smaller than a slice"
    assert be.folds >= 2 * (world - 1)
    fb, fe = bloom_byte_range(b, e, N_WORDS, N_BYTES)
    parts = [None] * world
    out = []
    be.dump_range(fb, fe - fb, out.append)
    dist.all_gather_object(parts, b"".join(out))
    assert b"".join(parts) == pack(want, 0, N_BYTES), "concatenated slices differ"
    print("OK", rank, b, e)
    dist.destroy_process_group()
''')


def _run(tmp_path, world, port):
    script = tmp_path / ("bloom_worker_%d.py" % world)
    script.write_text(WORKER % {"root": jfutil.ROOT, "m": 14014, "piece": 97})
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr",
                        "127.0.0.1", "--master-port", str(port), str(script)], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       timeout=300)
    out = r.stdout.decode()
    assert r.returncode == 0, out[-3000:]
    assert out.count("OK") == world, out[-3000:]


def test_bloom_reduce_scatter_world2_gloo(tmp_path):
    _run(tmp_path, 2, 29651)


def test_bloom_reduce_scatter_world3_gloo(tmp_path):
    _run(tmp_path, 3, 29652)


def test_bloom_slices_cover_the_counter_on_the_5_word_grid():
    from jellyfish_b200.distributed import bloom_byte_range, bloom_slices
    for m in (1, 79, 80, 81, 14014, 5600000, 10 ** 7 + 3):
        n_words, n_bytes = (m + 15) // 16, (m + 4) // 5
        for world in (1, 2, 3, 4, 7, 8):
            sl = bloom_slices(n_words, world)
            assert sl[0][0] == 0 and sl[-1][1] == n_words
            assert all(sl[r][1] == sl[r + 1][0] for r in range(world - 1))
            assert all(b % 5 == 0 or b == n_words for b, _ in sl)
            sizes = [e - b for b, e in sl]
            assert max(sizes) - min(sizes) <= 5
            br = [bloom_byte_range(b, e, n_words, n_bytes) for b, e in sl]
            assert br[0][0] == 0 and br[-1][1] == n_bytes
            assert all(br[r][1] == br[r + 1][0] for r in range(world - 1))
            assert all(fb % 16 == 0 or fb == n_bytes for fb, _ in br)


def _count_multi(*args):
    return subprocess.run([sys.executable, "-m", "jellyfish_b200.count_multi"] + list(args), cwd=jfutil.ROOT,
                          stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=120)


def test_count_multi_rejects_bloom_conflict_and_long_mers(tmp_path):
    fa = tmp_path / "x.fa"
    fa.write_text(">x\nACGT\n")
    r = _count_multi("-m", "21", "-s", "1M", "--bf-size", "1M", "--bc", str(fa), "-o", str(tmp_path / "o.jf"), str(fa))
    assert r.returncode != 0 and b"Switches [--bf-size] and [--bc] conflict" in r.stderr
    for sw in (["--bf-size", "1k"], ["--bc", str(fa)]):
        r = _count_multi("-m", "65", "-s", "1k", *sw, "-o", str(tmp_path / "o.jf"), str(fa))
        assert r.returncode != 0 and b"--bf-size and --bc take mer lengths up to 64" in r.stderr
    assert not (tmp_path / "o.jf").exists()
