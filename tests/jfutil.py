"""Helpers shared by the tests: locate binaries, run them, split jellyfish databases."""
import json
import os
import subprocess
import hashlib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
REF_JF = os.path.join(REF_DIR, "jellyfish")            # the unmodified reference, built by oracle/Makefile
ORACLE_C = os.path.join(REF_DIR, "jf_oracle")          # the independent C restatement
OUR_JF = os.path.join(ROOT, "jellyfish_b200", "lib", "jellyfish-b200")
LIB = os.path.join(ROOT, "jellyfish_b200", "lib", "libjfgpu.so")

SEMANTIC_KEYS = ("size", "key_len", "val_len", "max_reprobe", "reprobes", "counter_len", "format",
                 "canonical", "matrix1", "alignment")


def run(cmd, **kw):
    env = dict(os.environ, SOURCE_DATE_EPOCH="0")
    env.update(kw.pop("env", {}))
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=env, **kw)
    if r.returncode != 0:
        raise RuntimeError("command failed (%d): %s\nstdout: %s\nstderr: %s" % (
            r.returncode, " ".join(map(str, cmd)), r.stdout.decode(errors="replace")[-2000:],
            r.stderr.decode(errors="replace")[-2000:]))
    return r


def split_db(path):
    """-> (header dict, body bytes) of a jellyfish database."""
    with open(path, "rb") as f:
        data = f.read()
    hlen = int(data[:9])
    raw = data[9:9 + hlen].rstrip(b"\0")
    return json.loads(raw.decode()), data[9 + hlen:]


def semantic(header):
    return {k: header.get(k) for k in SEMANTIC_KEYS}


def md5(b):
    return hashlib.md5(b).hexdigest()


def records(header, body):
    """-> list of (key int, count int)"""
    kb = (header["key_len"] + 7) // 8
    cl = header["counter_len"]
    rec = kb + cl
    out = []
    for i in range(0, len(body) - rec + 1, rec):
        out.append((int.from_bytes(body[i:i + kb], "little"), int.from_bytes(body[i + kb:i + rec], "little")))
    return out


def subst(args, files):
    """'@name' in a case's switches stands for the path of that generated input (e.g. --if @multi2.fa)."""
    return [files[a[1:]] if a.startswith("@") else a for a in args]


def geometry(k, lsize, reprobe_limit=126):
    """The slot geometry table_setup (jellyfish_b200/csrc/jf_engine.cu) gives a table of 2^lsize slots requested: the
    table's own lsize (at most 2k, the key space), explicit key bits hb, clipped reprobe limit, reprobe field rbits, key
    field fb, key words, slot bits (320 = the wide form) and the in-slot counter bits cb.  slot_bits and cb are None where
    the key field fits no slot."""
    kbits = 2 * k
    if kbits < 64:
        lsize = min(lsize, kbits)
    hb = max(kbits - lsize, 0)
    limit = reprobe_limit if kbits > lsize else 0
    while limit >= 1 and limit * (limit + 1) // 2 >= (1 << lsize):        # reprobes[limit] < size
        limit -= 1
    rbits = (limit + 1).bit_length()
    fb = hb + rbits
    kw = 4 if k > 64 else 2 if k > 32 else 1
    if kw == 4:
        fb, sb = rbits + 1, 320
    else:
        sb = 32 if fb <= 22 else 64 if fb <= 56 else 128 if fb <= 127 else None
        if kw == 2 and sb == 32:
            sb = 64
    cb = None if sb is None else 64 - fb if sb in (64, 320) else 32 - fb if sb == 32 else 64 - max(fb - 64, 0)
    return {"k": k, "lsize": lsize, "hb": hb, "max_reprobe": limit, "rbits": rbits, "fb": fb, "kw": kw, "slot_bits": sb, "cb": cb}


def key_words(keys, k):
    """Python int keys -> uint64 array of shape (n, 64-bit words of a 2k-bit key)."""
    import numpy as np
    nw = (2 * k + 63) // 64
    return np.array([[(x >> (64 * w)) & 0xFFFFFFFFFFFFFFFF for w in range(nw)] for x in keys], dtype=np.uint64).reshape(-1, nw)


def positions(info, keys, k):
    """Original positions of Python int keys in a table described by HashCounter.info(), vectorised over the key words
    (RectangularBinaryMatrix::times, as hash_pos).  keys may also be an (n, words) uint64 array, as text_model gives."""
    import numpy as np
    words = keys if isinstance(keys, np.ndarray) else key_words(keys, k)
    size = info["size"]
    if info["matrix_identity"]:
        return words[:, 0] & np.uint64(size - 1)
    cols, c = info["matrix_columns"], info["matrix_c"]
    pos = np.zeros(len(words), np.uint64)
    for i in range(c):
        pos ^= ((words[:, i >> 6] >> np.uint64(i & 63)) & np.uint64(1)) * np.uint64(cols[c - 1 - i])
    return pos & np.uint64(size - 1)


def model_body(info, counts, k, ocl, lower=0, upper=(1 << 64) - 1):
    """binary/sorted body of {key: count}: records in (original position, key) order, ceil(2k/8) key bytes and ocl count
    bytes, counts clipped to 2^(8*ocl) - 1, only lower <= count <= upper."""
    keys = [x for x, c in counts.items() if lower <= c <= upper]
    pos = positions(info, keys, k).tolist() if keys else []
    kb, top = (2 * k + 7) // 8, (1 << (8 * ocl)) - 1
    return b"".join(x.to_bytes(kb, "little") + min(counts[x], top).to_bytes(ocl, "little")
                    for _, x in sorted(zip(pos, keys)))


def hash_pos(header, key):
    """Original position of a key: RectangularBinaryMatrix::times (bit i of the key selects columns[c-1-i],
    rectangular_binary_matrix.hpp:223-261) modulo the table size."""
    m = header["matrix1"]
    size = header["size"]
    if m.get("identity"):
        return key & (size - 1)
    cols, c = m["columns"], m["c"]
    h, i = 0, 0
    while key:
        if key & 1:
            h ^= cols[c - 1 - i]
        key >>= 1
        i += 1
    return h & (size - 1)
