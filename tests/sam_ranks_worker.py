"""torchrun worker of tests/test_gpu_split_sam.py: `count_multi` with every rank on device 0, the ranks joined by gloo
(NCCL takes one rank per device).  The ranks run the production path of several GPUs -- the split plan, the streamed
pieces, ShardedCounter.add_sam_pieces through the key exchange, the check after the count and its fall-back -- on one
H100.  Arguments: those of count_multi."""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from jellyfish_b200 import count_multi  # noqa: E402

argv = sys.argv[1:]
a = count_multi.parse_args(argv)
torch.cuda.set_device(0)
dist.init_process_group("gloo")
count_multi.run(a, argv, int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), 0)
