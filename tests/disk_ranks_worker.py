"""torchrun worker of tests/test_gpu_disk_multi.py: `count_multi` (its `main`, NCCL, one rank per GPU) with extra engine
keyword arguments for every rank's ShardedCounter, e.g. part_min_mb=1 so that small shards are filled region by region
and the count takes the record exchange.  Arguments: the keyword arguments as JSON, then those of count_multi."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from jellyfish_b200 import count_multi  # noqa: E402
from jellyfish_b200.distributed import ShardedCounter  # noqa: E402

extra = json.loads(sys.argv[1])
made = []


def make(*a, **kw):
    made.append(ShardedCounter(*a, **dict(kw, **extra)))
    return made[-1]


count_multi.ShardedCounter = make
count_multi.main(sys.argv[2:])
print("EXCHANGE rank %s %s" % (os.environ["RANK"], "records" if made[0].records is not None else "keys"))
