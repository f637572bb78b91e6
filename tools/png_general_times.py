"""The general PNG path per 3840x2160 frame and format (http_master.parse_png_general, usdu_png_decode_general_u8):

* parse: host time of parse_png_general (chunk walk, zlib inflate, filter-byte check), median of --reps;
* decode: device time of one usdu_png_decode_general_u8 launch for the frame (CUDA events), median of --reps;
* the card name and power limit, read in the same run.

Frames have random pixels and rows filtered with all five filters in turn, compressed at zlib level 1 (as fast
encoders write them), so the inflate times are an upper end for natural images of the same size.

    python tools/png_general_times.py [--reps 5] [--out results/png_general_times.json]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from collector_master_times import card  # noqa: E402
from __graft_entry__ import load_package  # noqa: E402

# name: (colour type, depth, interlace, PLTE entries)
FORMATS = {"rgb8_adam7": (2, 8, 1, None), "rgb16": (2, 16, 0, None), "rgb16_adam7": (2, 16, 1, None),
           "rgba16": (6, 16, 0, None), "grey16": (0, 16, 0, None), "grey1": (0, 1, 0, None),
           "pal8": (3, 8, 0, 256), "pal8_adam7": (3, 8, 1, 256), "pal4": (3, 4, 0, 16)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    load_package()
    import png_general_model as M
    from comfyui_distributed_b200 import http_master as hm
    H, W = 2160, 3840
    dev = torch.device("cuda")
    dst = torch.empty(H * W * 3, dtype=torch.uint8, device=dev)
    rows = {}
    for name, (color, depth, interlace, plte) in FORMATS.items():
        data = M.make_png(np.random.default_rng(1), color, depth, W, H, interlace, 1, 8, plte_entries=plte)
        parse, decode = [], []
        for i in range(a.reps + 1):
            t0 = time.perf_counter()
            info = hm.parse_png_general(data)
            t1 = time.perf_counter()
            dec = hm.PngDecoder(dev)
            dec.decode_general([(info, 0)], dst)
            torch.cuda.synchronize()
            if i:                                     # the first run warms up
                parse.append((t1 - t0) * 1e3)
                decode.append(dec.times()[1])
            dec.release()
        rows[name] = {"png_bytes": len(data), "filtered_bytes": info.raw_len,
                      "parse_ms": round(statistics.median(parse), 2), "decode_ms": round(statistics.median(decode), 3)}
        print(f"{name:12s} {len(data) / 1e6:7.1f} MB  parse {rows[name]['parse_ms']:8.2f} ms  "
              f"decode {rows[name]['decode_ms']:7.3f} ms", flush=True)
    out = {"card": card(), "frame": [H, W], "reps": a.reps, "formats": rows}
    print(json.dumps(out))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
