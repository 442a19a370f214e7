"""Tile census of the wgmma convolution engine over the convolutions of one network plan, from the engine's own geometry
(danet_conv_tc_geometry, the make_prob the kernels run), so that this model cannot drift from the kernel.  No GPU: the
plan is built on the CPU with the torch test double of the kernel layer, at batch 1, and every convolution's image
count is scaled to --batch (the plan's shapes are per image otherwise).

Per distinct convolution shape and in total, per network step:
  tiles        CTA tiles of the launch
  img/tile     images a tile stacks (small maps)
  eff          useful MACs / issued MACs (K padding, tile rows and columns past the map, stacking gaps)
  mma_share    share of all issued MACs
  tiles/unit   tiles per CTA work unit (danet_conv_tc_cta_geometry: exact mode pairs two tiles on one weight stream)
  w_GB, a_GB   weight and activation bytes copied from L2 into shared memory, per work unit times work units

    python tools/conv_census.py [--width 48] [--batch 64] [--precision exact] [--json FILE]
"""
import argparse
import collections
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def census(width=48, batch=64, precision="exact"):
    """{"shapes": [row, ...], "total": row} for the network's tensor-core convolutions at `batch`."""
    sys.path.insert(0, ROOT)
    import danet_b200
    from danet_b200 import _lib as L
    from oracle.net_ops import TorchEmulOps

    lib = L.load()
    net = danet_b200.build_synthetic_danet(width=width, seed=0, device="cpu", conv_algo="tc")
    plan = net.plan_for(1, "cpu", ops=TorchEmulOps())
    flags = 4 if precision == "exact" else 0
    count = collections.Counter()
    for s in plan.steps:
        if s.name != "conv_group":
            continue
        for cv in s.args[0]:
            d = cv["d"]
            count[(d["N"] * batch, d["H"], d["W"], d["Cin"], d["Cout"], d["ksize"], d["stride"], d["pad"], d["wsets"])] += 1
    rows = []
    out = (ctypes.c_int64 * 8)()
    cta = (ctypes.c_int64 * 4)()
    for key, n in count.items():
        N, H, W, Cin, Cout, k, st, pad, G = key
        d = L.ConvDesc(N, H, W, Cin, Cout, k, st, pad, G, 1, flags)
        L.check(lib.danet_conv_tc_geometry(ctypes.byref(d), ctypes.cast(out, ctypes.c_void_p)), "conv_tc_geometry")
        th, tw, tiles, nstack, products, macs_tile, a_tile, b_tile = list(out)
        L.check(lib.danet_conv_tc_cta_geometry(ctypes.byref(d), ctypes.cast(cta, ctypes.c_void_p)), "conv_tc_cta_geometry")
        per_unit, units, b_unit, a_unit = list(cta)
        Ho, Wo = (H + 2 * pad - k) // st + 1, (W + 2 * pad - k) // st + 1
        useful = N * Ho * Wo * Cout * Cin * k * k
        rows.append({"shape": "%dx%dx%d %d->%d %dx%d/s%d ws%d" % (N, H, W, Cin, Cout, k, k, st, G), "count": n,
                     "tile": "%dx%d" % (th, tw), "tiles": tiles * n, "img_per_tile": nstack,
                     "useful_macs": useful * n, "issued_macs": macs_tile * tiles * n, "products": products,
                     "eff": useful / float(macs_tile * tiles), "tiles_per_unit": per_unit, "units": units * n,
                     "w_bytes": b_unit * units * n, "a_bytes": a_unit * units * n})
    issued = sum(r["issued_macs"] for r in rows)
    for r in rows:
        r["mma_share"] = r["issued_macs"] / float(issued)
    rows.sort(key=lambda r: -r["issued_macs"])
    total = {"shape": "total", "count": sum(r["count"] for r in rows), "tiles": sum(r["tiles"] for r in rows),
             "units": sum(r["units"] for r in rows),
             "useful_macs": sum(r["useful_macs"] for r in rows), "issued_macs": issued,
             "w_bytes": sum(r["w_bytes"] for r in rows), "a_bytes": sum(r["a_bytes"] for r in rows)}
    total["eff"] = total["useful_macs"] / float(issued)
    return {"width": width, "batch": batch, "precision": precision, "shapes": rows, "total": total}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--width", type=int, default=48)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--precision", choices=("exact", "fast"), default="exact")
    ap.add_argument("--json", default=None, help="also write the census here")
    args = ap.parse_args()
    c = census(args.width, args.batch, args.precision)
    print("%-36s %5s %7s %8s %6s %6s %7s %9s %8s %8s" % ("shape", "convs", "tile", "tiles", "img/t", "t/unit", "eff",
                                                          "mma_share", "w_GB", "a_GB"))
    for r in c["shapes"] + [c["total"]]:
        print("%-36s %5d %7s %8d %6s %6s %7.3f %9s %8.2f %8.2f" % (
            r["shape"], r["count"], r.get("tile", ""), r["tiles"], r.get("img_per_tile", ""), r.get("tiles_per_unit", ""), r["eff"],
            "%.1f%%" % (100 * r.get("mma_share", 1.0)), r["w_bytes"] / 1e9, r["a_bytes"] / 1e9))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(c, f, indent=1)


if __name__ == "__main__":
    main()
