"""fp64-pipe probes (fastfp_fp64_peak kinds): 1 DMMA m16n8k4 peak (the sweep's shape), 19 / 20 / 21 DMMA m8n8k4 /
m16n8k8 / m16n8k16 peaks, 0 DFMA peak, 2 m8n8k4 + DFMA interleaved in one warp, 9/10/11 the m8n8k4 consumer tile (9x2
blocks, fragments from shared memory) with 2/4/1 warps per sub-partition, 23/24 the m16n8k4/k8 consumer tile, 13-15
warp-specialised m8n8k4 + DFMA mixes, 22 the same on m16n8k4 (8 MMA warps + 16 DFMA warps of 16 chains), 25 the same
mix at the m <= 80 sweep's split (8 MMA warps + 8 DFMA warps of 4 chains), 16 legacy INT8 mma.sync (T(FL)OP/s = 2 x MAC/s).
Prints TFLOP/s and ms."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fastfp_b200 import _cabi
for k in (int(a) for a in sys.argv[1:]) if len(sys.argv) > 1 else (1, 19, 20, 21, 0, 2, 9, 23, 24, 13, 14, 15, 22, 25, 16):
    _cabi.fp64_peak(k, 2000)
    print(k, _cabi.fp64_peak(k, 20000))
