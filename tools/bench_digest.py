"""Print the figures of a bench.py JSON line that matter when reading a log tail.
usage: python tools/bench_digest.py bench.json"""
import json
import sys


def r(v, n=1):
    return round(v, n) if isinstance(v, float) else v


def main():
    try:
        a = json.load(open(sys.argv[1]))
    except Exception as ex:
        print("bench parse failed:", ex)
        return
    print("value", r(a["value"]), a["dtype"], "ms/step", r(a["ms_per_step"], 2), "e2e", r(a["e2e"]["value"]), "launches", a["gpu_launches"],
          "n_gpus", a["n_gpus"], "host_ms", r(a.get("host_ms_per_step", 0.0), 2), "graph_replays", a.get("graph_replays"), "clocks", a.get("clocks"))
    rf = a.get("roofline")
    if rf:
        print("K1 roofline", {k: r(rf[k], 4) for k in ("frac", "achieved", "ms", "ms_single_launch_event_pair", "samples_per_launch", "unoccluded_gbs") if k in rf})
    if "roofline_step" in a:
        print("step tensor frac", r(a["roofline_step"]["frac"], 3))
    k = a.get("kernels", {})
    print("kernels_total_ms", a.get("kernels_total_ms"))
    for n, v in list(k.items())[:14]:
        print("   %-18s %8.3f ms  share %.3f  %s" % (n, v["ms"], v["share"], v.get("frac_of_hbm_peak", v.get("frac_of_bf16_peak"))))
    for key in ("scan", "patchcleanser_eval", "cpu_baseline", "value_scan_amortised"):
        if key in a:
            print(key, {q: r(w, 2) for q, w in a[key].items() if q != "note"} if isinstance(a[key], dict) else r(a[key]))
    for name, leg in a.get("legs", {}).items():
        print("leg", name, {q: (r(w, 2) if not isinstance(w, dict) else {a: r(b, 3) for a, b in w.items()}) for q, w in leg.items() if q not in ("kernels", "config")})
        if "kernels" in leg:
            for n, v in list(leg["kernels"].items())[:10]:
                print("   %-18s %8.3f ms  share %.3f  %s" % (n, v["ms"], v["share"], v.get("frac_of_hbm_peak", v.get("frac_of_bf16_peak"))))


if __name__ == "__main__":
    main()
