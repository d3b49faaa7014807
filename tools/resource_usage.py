#!/usr/bin/env python
"""(CPU) Registers / stack / static shared memory of every kernel of libkdb200.so (cuobjdump --dump-resource-usage):

    python tools/resource_usage.py > resource_usage.txt
"""
import re
import subprocess
from pathlib import Path

LIB = Path(__file__).resolve().parents[1] / "k-diffusion_b200" / "k_diffusion" / "_lib" / "libkdb200.so"


def main():
    text = subprocess.run(["cuobjdump", "--dump-resource-usage", str(LIB)], check=True, capture_output=True, text=True).stdout
    rows, name = [], None
    for line in text.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", line)
        if m and name:
            rows.append((name,) + tuple(int(v) for v in m.groups()))
            name = None
    names = subprocess.run(["c++filt"], input="\n".join(r[0] for r in rows), capture_output=True, text=True).stdout.split("\n")
    print("cuobjdump --dump-resource-usage libkdb200.so (sm_90a): registers per thread, stack bytes (spills / local arrays), static shared bytes.")
    print("Dynamic shared memory (the TMA-staged tiles of the tensor-core kernels) is requested at launch and is not listed here; SHARED = 1024 is the")
    print("1 KiB the CUDA 12.9 runtime reserves per CTA on sm_90.  STACK is the frame size (by-value parameter structs, trap paths of the mbarrier")
    print("time-outs, small local arrays), not a spill count.  `-Xptxas -v` (round 2 build) reports spills for 7 of the 101 kernels only:")
    print("gemm_tc_kernel<64,3> 8 B; ffn_fused_kernel 48 B stores / 116 B loads; attn_pipe_kernel variants 28-140 B stores / 108-176 B loads")
    print("(register cap 168 at 320 threads per CTA); every other kernel 0 bytes.  In ffn_fused_kernel no local load / store lies between the")
    print("first and the last MUFU.TANH of the GEGLU loop (SASS lines 1293-2079 of 4805): the spilled values are per-chunk loop state.\n")
    print(f"{'kernel':<72} {'REG':>4} {'STACK':>6} {'SHARED':>7}")
    for (_, reg, stack, shared, _local), d in zip(rows, names):
        d = re.sub(r"\((?:anonymous namespace|int|bool)\)", "", d)
        d = re.sub(r"\(.*", "", d).replace("::::", "::").replace("void ", "")
        print(f"{d[:72]:<72} {reg:>4} {stack:>6} {shared:>7}")
    spilled = [r for r in rows if r[2] > 0]
    print(f"\n{len(rows)} kernels; with a stack frame: {len(spilled)}")


if __name__ == "__main__":
    main()
