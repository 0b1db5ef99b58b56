"""Top stall sites of a kernel from an .ncu-rep captured with --import-source on (SASS view of the source page).

    python tools/ncu_hotspots.py bench_out/prof_gemm_pair8192.ncu-rep [N]
"""
import csv
import subprocess
import sys


def main(path, top=25):
    raw = subprocess.run(["ncu", "-i", path, "--page", "source", "--csv"], capture_output=True, text=True, check=True).stdout
    rows = list(csv.reader(raw.splitlines()))
    kernel, hdr, body = None, None, []
    out = []
    for r in rows:
        if r and r[0] == "Kernel Name":
            if kernel and body:
                out.append((kernel, hdr, body))
            kernel, hdr, body = r[1], None, []
        elif r and r[0] == "Address":
            hdr = r
        elif hdr and len(r) == len(hdr):
            body.append(r)
    if kernel and body:
        out.append((kernel, hdr, body))
    for kernel, hdr, body in out:
        i_src, i_all, i_not = hdr.index("Source"), hdr.index("Warp Stall Sampling (All Samples)"), hdr.index("Warp Stall Sampling (Not-issued Samples)")
        i_ex = hdr.index("Instructions Executed")
        total = sum(int(r[i_all] or 0) for r in body) or 1
        print(f"## {kernel[:110]}\n   {len(body)} SASS instructions, {total} stall samples\n")
        print("| samples | % | not issued | executed | SASS |\n|---|---|---|---|---|")
        for r in sorted(body, key=lambda r: -int(r[i_all] or 0))[:top]:
            print(f"| {r[i_all]} | {100 * int(r[i_all] or 0) / total:.1f} | {r[i_not]} | {r[i_ex]} | `{r[i_src].strip()}` |")
        print()


if __name__ == "__main__":
    main(sys.argv[1], int(sys.argv[2]) if len(sys.argv) > 2 else 25)
