"""Dominant GEMM launch of the bench step under ncu (run on a GPU):

    ncu --metrics dram__bytes_read.sum,dram__bytes_write.sum,gpu__time_duration.sum,sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active \
        --clock-control none -k regex:gemm_bf16_wgmma --csv --log-file bench_out/gemm_dram_bytes.csv python tools/prof_gemm.py

-> copy to profiles/rNN_gemm_dram_bytes.csv; bench.py reads roofline.traffic from the LAST launch in that file.
Shape = gate|up projection of a 64-crop frontier batch with the shared-prefix KV active (283 rows per crop): M = 18112, N = 22016
(gate/up interleaved, SwiGLU epilogue), K = 4096.  Algorithmic bytes = A 148.4 MB + W 180.4 MB + out 398.8 MB = 727.5 MB."""
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from vstar_b200 import ops  # noqa: E402

BF = torch.bfloat16
M, N, K = 64 * 283, 22016, 4096
a = torch.randn(M, K, device="cuda").to(BF)
w = (torch.randn(N, K, device="cuda") / math.sqrt(K)).to(BF)
out = torch.empty(M, N // 2, dtype=BF, device="cuda")
from vstar_b200 import _lib  # noqa: E402

# sweep (env PROF_GEMM_SWEEP=1): every hint mask x band height, 2 launches each; otherwise 3 launches of the shipped default
if os.environ.get("PROF_GEMM_SWEEP"):
    k = 0
    for gm in (16, 24, 8):
        _lib.call("vsb_gemm_set_group_m", gm)
        for mask in (0, 1, 4, 5, 8, 9, 12, 13):
            _lib.call("vsb_gemm_set_l2_hints", mask)
            for _ in range(2):
                ops.gemm(a, w, out=out, epilogue=ops.EPI_SWIGLU)
            torch.cuda.synchronize()
            print(f"launches {k}-{k + 1}: group_m={gm} hint_mask={mask}")
            k += 2
else:
    for _ in range(3):
        ops.gemm(a, w, out=out, epilogue=ops.EPI_SWIGLU)
    torch.cuda.synchronize()
print("algorithmic bytes", 2 * (M * K + N * K + M * N // 2))
