"""Time the convolution kernel alone on every shape of the PVCNN2 prior step (B=32):
python tools/bench_convs.py  -> table + JSON lines (CUDA events via lion_bench_conv).

Next to each time: the operand bytes the launch moves from L2 into shared memory (operand_bytes) and the rate that
makes -- the weight slabs every work item streams, and the activation windows of its tiles -- and the shared-memory
rings of the launch: taps per weight stage (9 = whole slabs, 3 = 3-tap parts, 1 = 1x1) and the depth of the
activation ring.  WHOLE_SLABS=1 makes every 3x3x3 launch stream whole weight slabs (same outputs; for comparisons)."""
import ctypes as C
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from lion_b200 import _lib as L

B = int(os.environ.get("B", "32"))
SHAPES = [  # (ntaps, cin, cout, r_or_rows, launches per step, label)
    (27, 4, 32, 32, 1, "sa0.0 conv1"), (27, 32, 32, 32, 3, "sa0.x conv"), (27, 128, 64, 16, 1, "sa1.0 conv1"),
    (27, 64, 64, 16, 1, "sa1.0 conv2"), (27, 192, 128, 8, 1, "sa2.0 conv1"), (27, 128, 128, 8, 13, "r=8 128->128"),
    (27, 128, 128, 16, 4, "fp2 r=16"), (27, 64, 64, 32, 4, "fp3 r=32"),
    (1, 36, 32, 32768, 1, "SA0 mlp0"), (1, 32, 64, 32768, 1, "SA0 mlp1"), (1, 68, 64, 8192, 1, "SA1 mlp0"),
    (1, 64, 128, 8192, 1, "SA1 mlp1"), (1, 196, 128, 2048, 1, "fp3 mlp0"), (1, 128, 128, 2048, 1, "fp3 mlp1"),
    (1, 64, 384, 1024, 1, "attn qkv"),
]
ONLY = os.environ.get("ONLY")  # e.g. ONLY="fp3 r=32" to time one shape (ncu captures)
if ONLY:
    SHAPES = [s for s in SHAPES if s[5] == ONLY]
if os.environ.get("TAPS"):           # TAPS=1 -> only the 1x1 shapes, TAPS=27 -> only the 3x3x3 ones
    SHAPES = [s for s in SHAPES if s[0] == int(os.environ["TAPS"])]


def _tiles_per_item(nt):
    return 4 if nt <= 32 else (2 if nt <= 64 else 1)


def _block_row(k, rp, nzb, npl):
    x, rem = divmod(k, npl)
    yb, zb = divmod(rem, nzb)
    return ((x + 1) * rp + 1 + 8 * yb) * rp + 1 + 8 * zb


def operand_bytes(ntaps, cin, cout, r_or_rows, B, num_sms, l2_bytes):
    """(work items, weight bytes, activation bytes) one launch of the tensor-core convolution reads from L2, from the
    tiling of conv_tc_prepare / conv_tc_run (csrc/conv_tc.cu): every item streams its n-tile's nchunk x ntg weight slabs
    once, and every tile the activation window of each slab.  Windows are counted whole: the clipped last window of a
    shape and skipped all-zero windows of a sparse input are not subtracted."""
    nt = cout if cout < 128 else 128
    n_nt, kg_all = cout // nt, cin // 4
    kg = 4 if (ntaps == 27 and nt > 64) else 8
    if kg_all < kg:
        kg = 2 if kg_all <= 2 else (4 if kg_all <= 4 else 8)
    nchunk, ntg, tpg = -(-kg_all // kg), (3 if ntaps == 27 else 1), (9 if ntaps == 27 else 1)
    b_stage = tpg * kg * nt * 16
    if ntaps == 27 and nt == 128:                     # interior 8 x 8 blocks, groups of 2 or 4 per item
        r, rp = r_or_rows, r_or_rows + 2
        nzb = -(-r // 8)
        npl = nzb * nzb
        nblk = r * npl

        def window(ib):
            return max(_block_row(min(f + ib, nblk) - 1, rp, nzb, npl) - _block_row(f, rp, nzb, npl) + 9 * rp + 10
                       for f in range(0, nblk, ib))
        fixed = 128 * 4 + 8 * 2 * nt * 4 + 64 * 8 + 128 + 1024
        four = (n_nt * B * -(-nblk // 4) >= num_sms
                and (227 * 1024 - fixed - 2 * b_stage) // (kg * window(4) * 16) >= 3)
        ib = 4 if four else 2
        stage_rows = window(ib)
        ntile, G, rows = -(-nblk // ib), 1, rp ** 3
    else:                                             # 128-row tiles, up to G per item
        rp = r_or_rows + 2 if ntaps == 27 else 0
        rows = rp ** 3 if ntaps == 27 else r_or_rows
        span = r_or_rows * rp * rp if ntaps == 27 else r_or_rows
        stage_rows = 128 + (2 * (rp + 1) if ntaps == 27 else 0)
        ntile, G = -(-span // 128), _tiles_per_item(nt)
    U = n_nt * B * ntile
    per_cta = -(-U // num_sms)
    grid = -(-U // per_cta)
    sched1 = ntaps == 27 and B * kg_all * rows * 16.0 > 1.6 * l2_bytes
    q, n_p = divmod(U, grid)
    m = -(-(q + (1 if n_p else 0)) // G)
    items = 0
    for i in range(grid):
        u, u_end = U * i // grid, U * (i + 1) // grid
        if sched1:                                    # one item per non-empty round (one n-tile: no cuts)
            items += min(u_end - u, m)
            continue
        while u < u_end:                              # a contiguous range cut into evenly sized items per n-tile
            run = min(u_end - u, B * ntile - u % (B * ntile))
            k2 = -(-run // G)
            u += -(-run // k2)
            items += 1
    slabs = nchunk * ntg
    return items, items * slabs * b_stage, U * slabs * kg * stage_rows * 16


def a_ring(ntaps, cin, cout, r_or_rows, B, num_sms, tps):
    """depth of the activation ring beside weight stages of tps taps (conv_tc_run's ring(), no side-stream cap)"""
    nt = cout if cout < 128 else 128
    kg_all = cin // 4
    kg = 4 if (ntaps == 27 and nt > 64) else 8
    if kg_all < kg:
        kg = 2 if kg_all <= 2 else (4 if kg_all <= 4 else 8)
    tpg = 9 if ntaps == 27 else 1
    fixed = 128 * 4 + 8 * 2 * nt * 4 + (8 * 2 * nt * 4 if tpg == 1 else 0) + 64 * 8 + 128 + 1024
    stage_b = tps * kg * nt * 16
    if ntaps == 27 and nt == 128:
        r, rp = r_or_rows, r_or_rows + 2
        nzb = -(-r // 8)
        nblk = r * nzb * nzb
        slab = 9 * kg * nt * 16

        def window(ib):
            return max(_block_row(min(f + ib, nblk) - 1, rp, nzb, nzb * nzb) - _block_row(f, rp, nzb, nzb * nzb) + 9 * rp + 10
                       for f in range(0, nblk, ib))
        four = (cout // nt) * B * -(-nblk // 4) >= num_sms and (227 * 1024 - fixed - 2 * slab) // (kg * window(4) * 16) >= 3
        stage_a = kg * window(4 if four else 2) * 16
    else:
        stage_a = kg * (128 + (2 * (r_or_rows + 3) if ntaps == 27 else 0)) * 16
    b_stages = 2 if tps == tpg else 4
    if ntaps == 27 and nt == 128 and tps == tpg:
        while b_stages < 4 and (227 * 1024 - fixed - (b_stages + 1) * stage_b) // stage_a >= max(4, b_stages + 1):
            b_stages += 1
    return min(16, (227 * 1024 - fixed - b_stages * stage_b) // stage_a)


torch.cuda.init()
L.check(L.lib().lion_ctx_set_conv_whole_slabs(L.ctx(), 1 if os.environ.get("WHOLE_SLABS") == "1" else 0), "whole slabs")
ITERS = int(os.environ.get("ITERS", "10"))      # ITERS=3000 CLOCKS=1: long enough for nvidia-smi to see the clock under load


def sample_clocks(stop, rows):
    import subprocess
    p = subprocess.Popen(["nvidia-smi", "-i", "0", "--query-gpu=clocks.sm,power.draw", "--format=csv,noheader,nounits", "-lms", "50"],
                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
    for line in p.stdout:
        rows.append([float(c) for c in line.split(",")])
        if stop.is_set():
            break
    p.terminate()


props = torch.cuda.get_device_properties(0)
tot = 0.0
for nt, ci, co, r, n, label in SHAPES:
    ms, fl = C.c_float(), C.c_double()
    rows, stop, th = [], None, None
    if os.environ.get("CLOCKS"):
        import threading
        stop = threading.Event()
        th = threading.Thread(target=sample_clocks, args=(stop, rows), daemon=True)
        th.start()
    L.check(L.lib().lion_bench_conv(L.ctx(), nt, ci, co, r, B, ITERS, 2, C.byref(ms), C.byref(fl), L.stream()), label)
    tf = fl.value / (ms.value * 1e-3) / 1e12
    tot += ms.value * n
    items, wb, ab = operand_bytes(nt, ci, co, r, B, props.multi_processor_count, props.L2_cache_size)
    tps = L.lib().lion_ctx_last_conv_stage_taps(L.ctx())
    rec = {"shape": label, "ntaps": nt, "cin": ci, "cout": co, "r_or_rows": r, "B": B, "ms": round(ms.value, 4),
           "tflops_algorithmic": round(tf, 1), "launches_per_step": n, "items": items, "weight_gb": round(wb / 1e9, 3),
           "activation_gb": round(ab / 1e9, 3), "weight_share": round(wb / (wb + ab), 2),
           "l2_to_smem_gbs": round((wb + ab) / (ms.value * 1e-3) / 1e9), "taps_per_weight_stage": tps,
           "a_stages": a_ring(nt, ci, co, r, B, props.multi_processor_count, tps)}
    if th is not None:
        stop.set()
        th.join(timeout=2)
        hot = sorted(x[0] for x in rows if x[1] > 300) or [x[0] for x in rows]
        rec["sm_mhz_under_load_median"] = hot[len(hot) // 2] if hot else None
        rec["power_w_max"] = max((x[1] for x in rows), default=None)
        rec["clock_samples"] = len(hot)
    print(json.dumps(rec))
print(json.dumps({"sum_ms_per_step_listed": round(tot, 3)}))
