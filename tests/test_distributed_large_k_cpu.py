"""CPU test (gloo, world_size 2) of the key exchange with four-word keys (k > 64): bucket -> count exchange -> uneven
all-to-all -> owner-side insertion must deliver every 32-byte key whole to its owner.  The device kernels are replaced by
a numpy backend behind the `RouteBackend` seam."""
import os
import subprocess
import sys
import textwrap

import jfutil

WORKER = textwrap.dedent('''
    import os, sys
    import numpy as np, torch, torch.distributed as dist
    sys.path.insert(0, %(root)r)
    from jellyfish_b200.distributed import RouteBackend, exchange_and_insert

    def owner(key, world):
        # every word decides: a key that arrived shifted or torn would land in the wrong table or not match
        return int((key[0] ^ (key[1] >> 3) ^ (key[2] >> 7) ^ (key[3] >> 11)) %% world)

    class NumpyBackend(RouteBackend):
        """keys: rows of 4 int64 words; "table" = python dict keyed by the 4-tuple"""
        key_words = 4
        def __init__(self, world): self.world = world; self.table = {}
        def extract_route(self, keys_in, begin, end, keys, capacity, counts):
            own = np.array([owner(k, self.world) for k in keys_in], dtype=np.int64) if len(keys_in) else np.zeros(0, np.int64)
            for d in range(self.world):
                mine = keys_in[own == d]
                keys[d, :mine.size] = torch.from_numpy(mine.reshape(-1).copy())
                counts[d] = len(mine)
        def insert_keys(self, keys, n):
            for row in keys[:n * 4].view(-1, 4).tolist():
                t = tuple(row)
                self.table[t] = self.table.get(t, 0) + 1

    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dist.init_process_group("gloo")
    rng = np.random.default_rng(200 + rank)
    # keys both ranks draw from (the same seed), so that owners receive the same key from both sides
    pool = np.random.default_rng(7).integers(-(1 << 62), 1 << 62, size=(300, 4), dtype=np.int64)
    be = NumpyBackend(world)
    cap = 3000
    send = torch.zeros((world, cap * 4), dtype=torch.int64); recv = torch.zeros((world, cap * 4), dtype=torch.int64)
    counts = torch.zeros(world, dtype=torch.int64)
    all_mine = []
    for rnd in range(3):                      # ragged rounds, one of them empty on rank 1
        n = 0 if (rank == 1 and rnd == 1) else int(rng.integers(1, 2500))
        keys_in = pool[rng.integers(0, len(pool), size=n)]
        all_mine.append(keys_in)
        counts.zero_()
        be.extract_route(keys_in, True, True, send, cap, counts)
        exchange_and_insert(be, world, send, counts, cap, recv)
    gathered = [None] * world
    dist.all_gather_object(gathered, np.concatenate(all_mine).tolist())
    expect = {}
    for lst in gathered:
        for k in lst:
            if owner(k, world) == rank:
                t = tuple(k)
                expect[t] = expect.get(t, 0) + 1
    assert be.table == expect, "rank %%d: table differs" %% rank
    assert all(owner(k, world) == rank for k in be.table)
    assert len(expect) > 10
    print("OK", rank, sum(be.table.values()))
    dist.destroy_process_group()
''')


def test_exchange_four_word_keys_world2_gloo(tmp_path):
    script = tmp_path / "worker4.py"
    script.write_text(WORKER % {"root": jfutil.ROOT})
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", MASTER_PORT="29633")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                        "--master-port", "29633", str(script)], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=300)
    out = r.stdout.decode()
    assert r.returncode == 0, out[-3000:]
    assert out.count("OK") == 2, out[-3000:]


def test_default_batch_of_four_word_keys():
    """The key exchange's three buffers stay near 8 GB for four-word keys; k <= 64 keeps its 256 MB batches."""
    from jellyfish_b200.distributed import default_batch_bytes
    assert default_batch_bytes(21) == default_batch_bytes(64) == 256 << 20
    assert default_batch_bytes(65) == default_batch_bytes(128) == 64 << 20
    per_buffer = default_batch_bytes(100) * 1.25 * 4 * 8
    assert 3 * per_buffer < 9 << 30
