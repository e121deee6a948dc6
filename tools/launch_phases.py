"""Attribute every launch of one training step to the library kernel it follows.

Input: the ncu launch list of bench.py's timed region (`ncu --metrics gpu__time_duration.sum --clock-control none
--profile-from-start off --csv --log-file launches.csv python bench.py ...`).  The step is a CUDA
graph, so the launch order is the capture order; the library's own kernels are used as phase markers and the torch
kernels between two markers ("glue": elementwise, reductions, index ops, cuBLAS calls of the backward) are summed.
Per-launch ncu times are cold-cache and serialised: read the SHARES, not the absolutes.

    python tools/launch_phases.py launches.csv > step_phase_attribution.txt
"""
import csv
import re
import sys

OWN = ("march_kernel", "app_mlp", "app_products", "composite_", "shade_", "density_", "valid_samples", "pack_",
       "unpack_", "heads_", "primary_", "scan_counts", "app_fill", "jitter_points", "epilogue_", "tail_", "adam_",
       "hits_prepare", "generate_rays")


def load(path):
    rows = list(csv.reader(open(path)))
    hdr = next(i for i, r in enumerate(rows) if r and r[0] == "ID")
    out = []
    for r in rows[hdr + 1:]:
        if len(r) > 14:
            t = float(r[14].replace(",", ""))
            out.append((r[4], r[8], t / 1e3 if r[13] == "ns" else t))
    return out


def short(name):
    name = re.sub(r"<unnamed>::|void |at::native::|native::", "", name)
    return re.sub(r"\(.*", "", name)[:48]


def main():
    launches = load(sys.argv[1])
    starts = [i for i, (n, _, _) in enumerate(launches) if "valid_samples_kernel<0>" in n]
    if len(starts) < 2:
        raise SystemExit("need at least two steps in the launch list")
    s, e = starts[0], starts[1]
    step = launches[s:e]
    total = sum(t for _, _, t in step)
    own_t = sum(t for n, _, t in step if any(o in n for o in OWN))
    print(f"# one step = launches [{s}, {e}) of {sys.argv[1]}: {len(step)} launches, {total / 1e3:.2f} ms under ncu")
    print(f"# library kernels {own_t / 1e3:.2f} ms ({100 * own_t / total:.0f} %), torch glue {(total - own_t) / 1e3:.2f} ms "
          f"({100 * (total - own_t) / total:.0f} %) in {sum(1 for n, _, _ in step if not any(o in n for o in OWN))} launches")
    print(f"# {'us':>9} {'share':>6}  kernel (grid)   |  glue launches that follow it: count, us, top kernels")
    i = 0
    while i < len(step):
        n, g, t = step[i]
        j = i + 1
        glue = {}
        gt = 0.0
        while j < len(step) and not any(o in step[j][0] for o in OWN):
            k = short(step[j][0])
            glue[k] = glue.get(k, 0.0) + step[j][2]
            gt += step[j][2]
            j += 1
        top = ", ".join(f"{k} {v:.0f}" for k, v in sorted(glue.items(), key=lambda kv: -kv[1])[:3])
        print(f"{t:10.1f} {100 * t / total:5.1f}%  {short(n)} {g}  |  {j - i - 1:3d} launches {gt:7.1f} us  {top}")
        i = j


if __name__ == "__main__":
    main()
