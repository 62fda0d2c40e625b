"""Summarise an `ncu --metrics gpu__time_duration.sum --csv` launch list into a markdown table (one train step).

Usage: python tests/probes/summarize_launches.py launches.csv "title" "command" [step_marker_kernel [step_index]]
The step is delimited by two consecutive launches of `step_marker_kernel` (e.g. input_pack: first kernel of a forward);
without a marker the whole file is one step."""
import collections
import csv
import re
import sys


def main():
    path, title, cmd = sys.argv[1:4]
    marker = sys.argv[4] if len(sys.argv) > 4 else None
    which = int(sys.argv[5]) if len(sys.argv) > 5 else 1
    rows = list(csv.reader(l for l in open(path) if l.startswith('"')))
    h = rows[0]
    ki, vi = h.index("Kernel Name"), h.index("Metric Value")
    body = rows[1:]
    if marker:
        idx = [i for i, r in enumerate(body) if marker in r[ki]]
        body = body[idx[which]:idx[which + 1]]
    agg, cnt = collections.Counter(), collections.Counter()
    for r in body:
        n = re.sub(r"\(.*", "", r[ki])
        n = re.sub(r"^void ", "", n)
        n = re.sub(r"<unnamed>::", "", n)
        agg[n] += float(r[vi].replace(",", ""))
        cnt[n] += 1
    tot = sum(agg.values())
    print(f"# {title}\n")
    print(f"Command: `{cmd}`")
    print("Per-launch times under ncu are serialised and cold-cache: compare SHARES, not absolutes.\n")
    print(f"Total device time of the step: {tot / 1e6:.1f} ms over {len(body)} launches.\n")
    print("| kernel | launches | total us | share | avg us |\n|---|---:|---:|---:|---:|")
    for n, v in agg.most_common(22):
        print(f"| `{n[:70]}` | {cnt[n]} | {v / 1e3:.0f} | {v / tot * 100:.1f}% | {v / 1e3 / cnt[n]:.1f} |")


if __name__ == "__main__":
    main()
