"""Phase clocks of the K == 128 GEMM kernel (co_gemm_tf32x3): where the producer and the consumers spend each row
tile.

Builds libcorollout.so with -DCO_GEMM_CLOCKS into its own directory (never the package's library), runs the GEMM at
the decoder-cache shape (M = 6 553 600, Nout = 640) and at an encoder shape (Nout = 384), and prints the mean cycles
per row tile of each phase over all CTAs:
  * producer: waiting on "empty" (the ring is full);
  * consumer warpgroup 0: waiting on "full" (A has not landed), load latency (TMA issue to the consumer passing
    "full"), A fragment reads + split + MMA issue, waiting for earlier MMA groups to retire, epilogue stores.

    python tools/gemm_phase_clocks.py [--out-dir DIR] [--json FILE]

The stamps cost a clock read per phase, so absolute cycles are a little above those of the shipped build.
"""
import argparse
import json
import os
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from rl4co_b200 import native  # noqa: E402

SLOTS = ["tiles", "producer_empty_wait", "load_latency", "full_wait", "issue", "retire_wait", "epilogue", "total"]
SHAPES = [(65536 * 100, 128, 640), (409600, 128, 384)]


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--out-dir", default=None, help="build directory of the diagnostic library (default: a temporary one)")
    p.add_argument("--json", default=None, help="also write the report here")
    a = p.parse_args()

    out_dir = a.out_dir or tempfile.mkdtemp(prefix="co_gemm_clocks_")
    native.LIB_PATH = native.build(extra_flags=["-DCO_GEMM_CLOCKS"], lib_path=os.path.join(out_dir, "libcorollout.so"))
    L = native.lib()
    L.co_gemm_clocks_set.argtypes = [native.c_void_p]

    dev = torch.device("cuda:0")
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    clk = torch.zeros(sms * 8, dtype=torch.int64, device=dev)  # one CTA per SM at most
    assert L.co_gemm_clocks_set(clk.data_ptr()) == 0  # before any launch: the kernel does not test the pointer
    rep = {"gpu": torch.cuda.get_device_name(dev), "shapes": []}
    for M, K, Nout in SHAPES:
        torch.manual_seed(0)
        x = torch.randn(M, K, device=dev)
        hi, lo = native.split_tf32(torch.randn(Nout, K, device=dev) / K ** 0.5)
        out = torch.empty(M, Nout, device=dev)
        for _ in range(2):  # warm-up, then the run whose stamps are kept
            clk.zero_()
            native.gemm_tf32x3(x, hi, lo, out=out)
        torch.cuda.synchronize()
        c = clk.view(sms, 8).cpu().double()
        c = c[c[:, 0] > 0]
        tiles = c[:, 0].sum().item()
        row = {"M": M, "K": K, "Nout": Nout, "ctas": int(c.shape[0]),
               "cycles_per_tile": {k: c[:, i].sum().item() / tiles for i, k in enumerate(SLOTS) if i > 0}}
        rep["shapes"].append(row)
        print(f"{rep['gpu']}: M={M} K={K} Nout={Nout}, {row['ctas']} CTAs, mean cycles per row tile")
        for k, v in row["cycles_per_tile"].items():
            print(f"  {k:20s} {v:9.1f}")
        del x, out
    if a.json:
        with open(a.json, "w") as f:
            json.dump(rep, f, indent=1)


if __name__ == "__main__":
    main()
