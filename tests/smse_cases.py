"""The sample_mse census cases shared by test_sample_mse_census_cpu.py (mutants) and test_sample_mse_census_gpu.py.

A case names its split count, not its head count: the GPU test picks BH from the device's SM count so that
smse_layout gives that nsplit (bh_for).  Head h of a case depends on (seed, h) only, so the first heads are the same
whatever BH is, and the CPU suite can run them at the same split count.
"""
import torch

# name, layout, ctx, F, P, D, dtype, n_rows, nsplit, hot, seed
CASES = [
    ("hy_p200_d128_n64_s3", "hy", 48, 6, 200, 128, torch.bfloat16, 64, 3, True, 1),
    ("hy_p256_d64_n127_s8_empty", "hy", 64, 5, 256, 64, torch.float16, 127, 8, True, 2),
    ("hy_p80_d64_n7_s2", "hy", 20, 9, 80, 64, torch.bfloat16, 7, 2, True, 3),
    ("wan_p180_d64_n1_s2", "wan", 0, 7, 180, 64, torch.float16, 1, 2, True, 4),
    ("wan_p600_d64_n128_s32_empty", "wan", 0, 7, 600, 64, torch.bfloat16, 128, 32, True, 5),
    ("cog_p260_d128_n9_s1", "cog", 40, 4, 260, 128, torch.float16, 9, 1, True, 6),
    ("cog_p80_d64_n8_s6_chunkcap", "cog", 20, 9, 80, 64, torch.bfloat16, 8, 6, True, 7),
    ("cog_p1350_d128_n63_s32_empty", "cog", 226, 3, 1350, 128, torch.bfloat16, 63, 32, True, 8),
    ("hy_p200_d128_n64_s3_census", "hy", 48, 6, 200, 128, torch.bfloat16, 64, 3, False, 9),
    ("wan_p600_d128_n9_s32_census_empty", "wan", 0, 7, 600, 128, torch.float16, 9, 32, False, 10),
    ("cog_p1350_d64_n64_s1_census", "cog", 226, 3, 1350, 64, torch.float16, 64, 1, False, 11),
    ("hy_p200_d64_n128_s3_census", "hy", 48, 6, 200, 64, torch.bfloat16, 128, 3, False, 12),
]


def pick_rows(lay, ctx, F, P, n, seed):
    """n sampled rows: the last row, frame and 128-row edges, text rows, random rows and (n >= 8) duplicates."""
    S = ctx + F * P
    V = F * P
    vid0 = ctx if lay == "cog" else 0
    special = [S - 1, vid0, vid0 + P - 1, vid0 + P, 127, 128, 255, 256, vid0 + V // 2, vid0 + (F - 1) * P]
    if ctx:
        special += [ctx - 1, 0] if lay == "cog" else [V, V + ctx - 1, V - 1]
    special = [r for r in dict.fromkeys(special) if 0 <= r < S]
    g = torch.Generator().manual_seed(seed)
    rnd = torch.randint(0, S, (n,), generator=g).tolist()
    rows = (special + rnd)[:n]
    if n >= 8:
        rows[-1] = rows[1]
        rows[-2] = rows[0]
    return torch.tensor(rows, dtype=torch.long)


def bh_for(nsplit, n_sms):
    """a head count at which smse_layout gives nsplit splits (before the n_chunks cap) on a device of n_sms SMs"""
    if nsplit >= 32:
        return max(1, n_sms // 33)
    if nsplit == 1:
        return n_sms // 2 + 1
    return n_sms // nsplit


def build(case, BH):
    from oracle import smse_census as sc

    name, lay, ctx, F, P, D, dt, n, nsplit, hot, seed = case
    rows = pick_rows(lay, ctx, F, P, n, seed)
    return sc.make_case(lay, ctx, F, P, D, BH, rows, hot=hot, seed=seed)
