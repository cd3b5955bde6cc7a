#!/usr/bin/env python
"""Per-shape table of a GO1_GEMM_TIMING_CSV dump (one PPO update): launches, total / mean microseconds, TFLOP/s, share.  The bf16 column
tells the operand paths apart: 0 TF32, 1 BF16 K-major (go1_gemm_bf16_ex), 2 BF16 in either major (go1_gemm_bf16_mn / _grouped, the products
of AC_Args.bf16_backward)."""
import collections, csv, sys


def main(path):
    rows = list(csv.DictReader(open(path)))
    agg = collections.OrderedDict()
    for r in rows:
        k = (r['M'], r['N'], r['K'], r['a_mn_major'], r['b_mn_major'], r['act'], r['num_extra'], r['splits'], r['kernel'], r['colsum'], r['n3'], r['heads'],
             r['problems'], r.get('bf16', '0'))
        a = agg.setdefault(k, [0, 0.0]); a[0] += 1; a[1] += float(r['us'])
    tot = sum(v[1] for v in agg.values())
    print(f"total {tot / 1e3:.2f} ms over {len(rows)} launches")
    print("M N K amn bmn act nex splits kern colsum n3 heads problems bf16 | n total_us avg_us TF/s share%")
    for k, v in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        M, N, K = int(k[0]), int(k[1]), int(k[2])
        fl = 2 * M * N * K
        if k[8].startswith('tail'):      # M rows of all problems through K1 -> N2 (-> N3), then each problem's head on its M / problems rows
            n3, heads, probs = int(k[10]), int(k[11]), int(k[12])
            fl = 2 * M * (K * N + N * n3) + 2 * (M // probs) * (n3 or N) * heads
        print(*k, '|', v[0], round(v[1]), round(v[1] / v[0], 1), round(fl / (v[1] / v[0]) / 1e6, 1), round(100 * v[1] / tot, 1))


if __name__ == "__main__":
    main(sys.argv[1])
