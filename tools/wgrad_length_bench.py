"""Per-call time of the weight-gradient GEMM (dc_gemm_wgrad_tf32x3, dc_unit_wgrad_routed) at c4's shapes (CUDA events),
plus the L2 traffic its accumulator flushes add.  One JSON line; the card's name and power limit are part of it.

    python tools/wgrad_length_bench.py [--iters 20] [--windows 7]

The accumulator flushes (gemm_tf32x3.cu, kWgFlush) send 64 KB of vector reductions per CTA into L2 for every flush after
the first (the first stores, as the partial always did); unit_dgrad_kernel's (kDgFlush) send its [128][13] partial, 6.7 KB.
Counted here from the shapes, not measured; FLUSH_ROWS and DG_FLUSH_TILES follow the two constants."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
from dotaclient_b200 import _lib, ops  # noqa: E402

FLUSH_ROWS = 128 * 32           # kWgFlush chunks of 32 rows
DG_FLUSH_TILES = 32             # kDgFlush
SHAPES = [("pre_rnn c4", "plain", 512, 896, 524288), ("w_ih c4", "plain", 2048, 512, 524288),
          ("unit16 c4", "routed", 128, 16, 524288), ("unit16 dgrad c4", "dgrad", 128, 16, 524288)]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        q = torch.cuda.get_device_name(0) + ", power limit not read"
    return q


def flush_l2_bytes(No, Ni, rows):
    """Extra bytes one call sends to L2: per CTA, a 64 KB reduction into its partial for every flush after the first."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tiles = ((No + 127) // 128) * ((Ni + 127) // 128)
    nsplit = max(1, sms // tiles)
    per_cta = -(-rows // nsplit)
    extra = max(0, -(-per_cta // FLUSH_ROWS) - 1)
    return tiles * nsplit * extra * 128 * 128 * 4


def dgrad_flush_l2_bytes(rows):
    """The same for dc_unit_dgrad_fused_mask: per CTA, a [128][13] reduction for every flush after the first."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    m_blocks = -(-rows // 128)
    grid = min(sms, m_blocks)
    tiles_per_cta = -(-m_blocks // grid)
    extra = max(0, -(-tiles_per_cta // DG_FLUSH_TILES) - 1)
    return grid * extra * 128 * 13 * 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--windows", type=int, default=7)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    lib, st = _lib.load(), _lib.stream_ptr()
    g = torch.Generator(device=dev).manual_seed(0)
    result = {"card": card(), "kernels": {}}
    for name, form, No, n, T in SHAPES:
        if form == "plain":
            dy, x = torch.randn(T, No, generator=g, device=dev), torch.randn(T, n, generator=g, device=dev)
            dw, db = torch.empty(No, n, device=dev), torch.empty(No, device=dev)
            fn = lambda: ops.gemm_wgrad_tf32x3(dy, x, dw_out=dw, db_out=db)  # noqa: E731
            rows, Ni = T, n
        elif form == "dgrad":
            d = torch.randn(T, 128, generator=g, device=dev)
            units = torch.randn(T * n, 12, generator=g, device=dev)
            w_b, b_b = torch.randn(128, 12, generator=g, device=dev) * 0.3, torch.randn(128, generator=g, device=dev) * 0.1
            w_t = torch.randn(128, 128, generator=g, device=dev) * 0.1
            am = torch.randint(0, n, (T, 128), generator=g, device=dev, dtype=torch.uint8)
            ws = torch.empty(int(lib.dc_unit_basic_bwd_workspace_bytes()), dtype=torch.uint8, device=dev)
            dw, db = torch.empty(128, 12, device=dev), torch.empty(128, device=dev)
            fn = lambda: _lib.check(lib.dc_unit_dgrad_fused_mask(  # noqa: E731
                d.data_ptr(), None, 128, am.data_ptr(), None, 0, None, w_t.data_ptr(), units.data_ptr(), None, w_b.data_ptr(),
                b_b.data_ptr(), T, n, dw.data_ptr(), db.data_ptr(), 0, ws.data_ptr(), st), "dgrad")
            rows, Ni = T * n, 128
        else:
            d = torch.randn(T, 128, generator=g, device=dev)
            basic = torch.relu(torch.randn(T * n, 128, generator=g, device=dev))
            am = torch.randint(0, n, (T, 128), generator=g, device=dev, dtype=torch.uint8)
            ws = torch.empty(int(lib.dc_gemm_wgrad_workspace_bytes(128, 128)), dtype=torch.uint8, device=dev)
            dw, db = torch.empty(128, 128, device=dev), torch.empty(128, device=dev)
            fn = lambda: _lib.check(lib.dc_unit_wgrad_routed(d.data_ptr(), None, 128, am.data_ptr(), basic.data_ptr(), T, n,  # noqa: E731
                                                             dw.data_ptr(), db.data_ptr(), ws.data_ptr(), st), "routed")
            rows, Ni = T * n, 128
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        times = []
        for _ in range(args.windows):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.iters):
                fn()
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1) / args.iters)
        times.sort()
        result["kernels"][name] = {"ms_median": times[len(times) // 2], "ms_min": times[0], "ms_max": times[-1],
                                   "flush_l2_mb": (dgrad_flush_l2_bytes(rows) if form == "dgrad" else flush_l2_bytes(No, Ni, rows)) / 1e6}
        del fn
        torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
