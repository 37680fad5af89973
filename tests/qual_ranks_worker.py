"""torchrun worker of tests/test_gpu_qual_count_multi.py: `count_multi` with every rank on device 0, the ranks joined by
gloo (NCCL takes one rank per device), and the key exchange's text per round cut down to BATCH bytes, so that the
exchange rounds of a whole file and the pieces of a share end inside the small test files.  The ranks run the production
path of several GPUs -- the split plan, the record-aligned pieces and rounds under -Q, the two passes of --if, the check
after the count and its fall-back -- on one H100.  Arguments: BATCH, then those of count_multi."""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from jellyfish_b200 import count_multi, distributed  # noqa: E402

batch = int(sys.argv[1])
argv = sys.argv[2:]
distributed.default_batch_bytes = lambda k: batch
a = count_multi.parse_args(argv)
torch.cuda.set_device(0)
dist.init_process_group("gloo")
count_multi.run(a, argv, int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), 0)
