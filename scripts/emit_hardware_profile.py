#!/usr/bin/env python
"""Turn the measured collective tables (scripts/bench_collectives.py JSON lines) into the hardware-profile JSONs the
reference Search Engine reads (SURVEY 8f-4; formats: galvatron/profile_hardware/hardware_configs/*.json, consumed by
galvatron/utils/config_utils.py:59-91,108-137):
    allreduce_bandwidth_1nodes_<N>gpus_per_node.json   {"allreduce_size_<n>_consec_<c>": bus GB/s}
    sp_time_1nodes_<N>gpus_per_node.json               {"allreduce_size_<n>_<MB>MB_time": ms, "all2all_size_<n>_<MB>MB_time": ms}
    p2p_bandwidth_1nodes_<N>gpus_per_node.json         {"pp_size_<n>": GB/s}
    overlap_coefficient.json                           {"overlap_coe": x}
NVSwitch gives strided and consecutive groups the same bandwidth, so consec_0 == consec_1.

    python scripts/emit_hardware_profile.py collectives_2gpu.jsonl [more.jsonl ...] --out <dir for search_strategy.py --hardware-dir>
"""
import argparse
import json
import math
import os


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("tables", nargs="+")
    ap.add_argument("--out", required=True)
    ap.add_argument("--gpus-per-node", type=int, default=8)
    opts = ap.parse_args()
    rows = []
    for path in opts.tables:
        for line in open(path):
            line = line.strip()
            if line.startswith("{"):
                rows.append(json.loads(line))
    by = {}
    for r in rows:
        by.setdefault((r["op"], r["p"]), []).append(r)
    os.makedirs(opts.out, exist_ok=True)
    N = opts.gpus_per_node
    ar, sp, p2p = {}, {}, {}
    sizes_mb = [1, 2, 4, 8, 16, 32, 64, 128, 256, 512, 1024]

    def interp(points, mb):
        """log-log interpolation of time(ms) over message size"""
        pts = sorted((r["bytes"] / 2 ** 20, r["ms"]) for r in points)
        if mb <= pts[0][0]:
            return pts[0][1]
        for (x0, y0), (x1, y1) in zip(pts, pts[1:]):
            if x0 <= mb <= x1:
                t = (math.log(mb) - math.log(x0)) / (math.log(x1) - math.log(x0))
                return math.exp(math.log(y0) + t * (math.log(y1) - math.log(y0)))
        (x0, y0), (x1, y1) = pts[-2], pts[-1]
        return y1 * mb / x1
    measured_p = sorted({p for (_, p) in by})
    for n in (2, 4, 8):
        src = n if n in measured_p else (max(measured_p) if measured_p else None)
        if src is None:
            continue
        arp = by.get(("all_reduce", src), [])
        a2a = by.get(("ulysses_all_to_all", src), [])
        if arp:
            big = max(arp, key=lambda r: r["bytes"])
            # reference unit: bus bandwidth GB/s (nccl-tests convention)
            for c in (0, 1):
                ar["allreduce_size_%d_consec_%d" % (n, c)] = big["busGBps"]
            for mb in sizes_mb:
                scale = (2 * (n - 1) / n) / (2 * (src - 1) / src)
                sp["allreduce_size_%d_%dMB_time" % (n, mb)] = interp(arp, mb) * scale
        if a2a:
            for mb in sizes_mb:
                scale = ((n - 1) / n) / ((src - 1) / src)
                sp["all2all_size_%d_%dMB_time" % (n, mb)] = interp(a2a, mb) * scale
        ag = by.get(("all_gather_cast", src), [])
        if ag:
            # one-direction peer stores between two GPUs, measured at p=2 (the all-gather's bus bandwidth there IS the pairwise
            # rate); NVSwitch gives every stage boundary the same link whatever the pipeline depth
            pair = by.get(("all_gather_cast", 2), ag)
            p2p["pp_size_%d" % n] = max(pair, key=lambda r: r["bytes"])["busGBps"]
    json.dump(ar, open(os.path.join(opts.out, "allreduce_bandwidth_1nodes_%dgpus_per_node.json" % N), "w"), indent=4)
    json.dump(sp, open(os.path.join(opts.out, "sp_time_1nodes_%dgpus_per_node.json" % N), "w"), indent=4)
    json.dump(p2p, open(os.path.join(opts.out, "p2p_bandwidth_1nodes_%dgpus_per_node.json" % N), "w"), indent=4)
    json.dump({"overlap_coe": 1.0}, open(os.path.join(opts.out, "overlap_coefficient.json"), "w"), indent=4)
    print("wrote", opts.out, "from ranks measured:", measured_p)


if __name__ == "__main__":
    main()
