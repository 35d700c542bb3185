"""Discrete-event model of the staged lock-step scheduler of k_encode_mbs (openh264_b200/csrc/enc_kernels.cu).

Why: on the GPU the kernel is bound by its dependency structure (much of the warp time waits at batch barriers), and scheduler variants cost GPU time to try.  This model replays the REAL
per-macroblock stage paths of the bench clip (recorded by the host build of the macroblock code,
tools/sim_data/mb_stage_paths_1080p.npy: bit s set = stage s ran; A=1, I=2, Bs=3, B=4, C=5) through the same
policy — one CTA per SM (132 on an H100), W warps each, a batch = up to W ready tasks of ONE stage, batch time = slowest task
(body + per-task overhead) + a per-batch overhead, later stages first, a full batch beats a partial one — with the recorded
stage costs (tools/enc_stats.py, see COST).

Variant `pull` models ENC_PULL (enc_kernels.cu, run_stages): a full batch of list A or Bs claims up to pull x W tasks, every
warp starts one, and each further task goes to the warp that becomes free first; every task notifies its dependants at its
own end, the batch ends when its last warp does.

usage: python tools/sched_sim.py [--streams 256] [--warps 24] [--variant base|dfill|dfull|half|patience|fastB|pull] [--pull 2]
"""
import argparse
import heapq
import os
import random

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
A, I, BS, B, C, D = 1, 2, 3, 4, 5, 6
# task body cycles (g_enc_stats), stage -> cycles: tools/enc_stats.py 256 with ENC_PULL = 1, P picture 5, on one H100 80GB HBM3
# (700 W power limit, 1,980 MHz); I = the stage-I task on the same card; D = deblocking as a task, a placeholder: in-loop
# deblocking is a separate kernel
COST = {A: 20200, BS: 15700, B: 131800, C: 235700, D: 11200, I: 206000}
# same run: per task, task wall (g_task_wall) minus body of stage A = fences, unpark / park, notifications (26.9 k - 20.2 k);
# per batch, the leader wait (what the workers waited for the claim: 1.72 G cycles over 142 k batches); the slowest-warp tail
# comes from the task spread.  The model then gives 38.6 ms where the GPU measured 39.0 ms (ENC_PULL = 1), and predicts pull 2
# at 36.2 ms and pull 3 at 35.2 ms, where the GPU measured 34.2 and 34.5 ms (DESIGN.md §7).
TASK_OVERHEAD = 6700
BATCH_OVERHEAD = 12000
MBW, MBH = 120, 68


def build_paths(n_streams, seed=1):
    paths = np.load(os.path.join(ROOT, "tools", "sim_data", "mb_stage_paths_1080p.npy"))
    rng = random.Random(seed)
    return [paths[rng.randrange(len(paths))] for _ in range(n_streams)]


def simulate(n_streams=256, warps=24, n_cta=132, variant="base", seed=1, cost=None, verbose=False, pull=2):
    cost = dict(COST if cost is None else cost)
    if variant == "fastB":
        cost[B] = int(cost[B] * 0.7)
    rng = random.Random(seed)
    paths = build_paths(n_streams, seed)
    n_mb = MBW * MBH
    total = n_streams * n_mb
    with_d = variant in ("dfill", "dfull")
    groups = 2 if variant == "half" else 1                 # lock-step groups per CTA
    gw = warps // groups
    dep = np.zeros(total, np.int8)
    depd = np.zeros(total, np.int8)
    queues = {k: [] for k in (A, BS, B, C, D)}
    heads = {k: 0 for k in queues}
    for s in range(n_streams):
        queues[A].append(s * n_mb)
    coded = deblocked = 0
    # event heap: (time, seq, group id, stage, [task ids])
    ev = []
    seq = 0
    idle = list(range(n_cta * groups))
    busy_cycles = {k: 0 for k in queues}
    batch_n = {k: 0 for k in queues}
    batch_tasks = {k: 0 for k in queues}
    group_time = 0                                          # sum over batches of (duration) = CTA-group-cycles busy
    now = 0
    order = [C, B, BS, A] + ([D] if with_d else [])

    def avail(k):
        return len(queues[k]) - heads[k]

    def next_stage(mask, stage):
        for s in (BS, B, C):
            if s > stage and (mask >> s) & 1:
                return s
        return 0

    def notify_d(si, x, y):
        did = si * n_mb + y * MBW + x
        depd[did] += 1
        if depd[did] == 1 + (x > 0) + (y > 0):
            queues[D].append(did)

    def finish(task, stage):
        nonlocal coded, deblocked
        si, mb = divmod(task, n_mb)
        y, x = divmod(mb, MBW)
        if stage == D:
            if x + 1 < MBW:
                notify_d(si, x + 1, y)
            if y + 1 < MBH:
                if x > 0:
                    notify_d(si, x - 1, y + 1)
                if x == MBW - 1:
                    notify_d(si, x, y + 1)
            deblocked += 1
            return
        nxt = next_stage(int(paths[si][mb]), stage)
        if nxt:
            queues[nxt].append(task)
            return
        coded += 1
        if x + 1 < MBW:
            dep[task + 1] += 1
            if dep[task + 1] == 1 + (y > 0):
                queues[A].append(task + 1)
        if y + 1 < MBH:
            if x > 0:
                dep[task + MBW - 1] += 1
                if dep[task + MBW - 1] == 1 + (x - 1 > 0):
                    queues[A].append(task + MBW - 1)
            if x == MBW - 1:
                dep[task + MBW] += 1
                if dep[task + MBW] == 1 + (x > 0):
                    queues[A].append(task + MBW)
        if with_d:
            if x > 0 and y > 0:
                notify_d(si, x - 1, y - 1)
            if x == MBW - 1 and y > 0:
                notify_d(si, x, y - 1)
            if y == MBH - 1 and x > 0:
                notify_d(si, x - 1, y)
            if x == MBW - 1 and y == MBH - 1:
                notify_d(si, x, y)

    def pick():
        """the leader's choice: (stage, n) or None"""
        best, best_avail = None, 0
        for k in order:
            a = avail(k)
            if variant == "dfill" and k == D:
                # deblocking only fills: take it when no coding task at all is ready (or coding is over)
                if best is None and a > 0:
                    return D, min(gw, a)
                continue
            if a >= gw:
                return k, min(a, pull * gw) if variant == "pull" and k in (A, BS) else gw
            if a > best_avail:
                best, best_avail = k, a
        if best is None:
            return None
        if variant == "patience" and best_avail < gw // 2 and len(ev) > 0:
            return None                                   # wait for the next completion instead of a thin batch
        return best, best_avail

    def dispatch():
        nonlocal seq, group_time
        while idle:
            c = pick()
            if c is None:
                return
            k, n = c
            g = idle.pop()
            tasks = queues[k][heads[k]:heads[k] + n]
            heads[k] += n
            # every warp notifies its dependants as soon as ITS task is done; the group is free after the slowest
            durs = [int(cost[k] * rng.uniform(0.85, 1.2) * (1.0 if k != B else rng.choice((1.0, 1.0, 1.0, 1.35)))) + TASK_OVERHEAD
                    for _ in tasks]
            # warp ends: a task more than the group's warps goes to the warp that is free first (only a pulled batch has those)
            free = [0] * min(n, gw)
            ends = []
            for d in durs:
                j = min(range(len(free)), key=free.__getitem__)
                free[j] += d
                ends.append(free[j])
            dur = max(free) + BATCH_OVERHEAD
            busy_cycles[k] += sum(durs)
            batch_n[k] += 1
            batch_tasks[k] += n
            group_time += dur
            for t, e in zip(tasks, ends):
                seq += 1
                heapq.heappush(ev, (now + e, seq, -1, k, t))
            seq += 1
            heapq.heappush(ev, (now + dur, seq, g, k, None))

    dispatch()
    while ev:
        now, _, g, k, task = heapq.heappop(ev)
        if g < 0:
            finish(task, k)
        else:
            idle.append(g)
        if idle:
            dispatch()
    assert coded == total and (not with_d or deblocked == total), (coded, deblocked, total)
    ms = now / 1.965e6
    res = {"variant": variant + (str(pull) if variant == "pull" else ""), "streams": n_streams, "warps": warps, "kernel_ms": round(ms, 2),
           "group_busy_frac": round(group_time / (now * n_cta * groups), 3),
           "warp_busy_frac": round(sum(busy_cycles.values()) / (now * n_cta * warps), 3),
           "fill": {k: round(batch_tasks[k] / max(1, batch_n[k]), 1) for k in queues if batch_n[k]}}
    return res


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=256)
    ap.add_argument("--warps", type=int, default=24)
    ap.add_argument("--variant", default="base")
    ap.add_argument("--pull", type=int, default=2, help="variant pull: claim up to this many warps' worth of A / Bs tasks")
    a = ap.parse_args()
    print(simulate(a.streams, a.warps, variant=a.variant, pull=a.pull))
