"""The host side and the per-kernel layouts of farthest point sampling (csrc/fps.cu) restated in Python.  No device is
needed.

- ``CTA_KERNELS`` / ``CLUSTER_KERNELS`` / ``BIG_KERNELS``: the three PN2_FPS_*_KERNELS lists, and ``INSTANCES``: every
  kernel the dispatcher can launch (family, P, T, PR, V), the global-scratch fallback included.
- ``plan_fps``: the planner: the single-CTA table, the cluster search with its co-residency rule, the cost model, and
  the decoding of a tuning override (``pn2_set_fps_config``): the chain in the two low bits of ``threads``, the PR rule,
  cluster -1 / -2.
- ``dispatch``: which instantiation a plan runs, or why the dispatcher refuses it.
- ``owner`` / ``stages``: where each kernel keeps point k (thread, CTA rank, register slot, search group, streamed or
  not), and for two tied points the stage of the kernel that decides between them.  Every kernel must pick the first
  tied point in the order (k mod 512, k); the stages are the places where a kernel can get that wrong.

The capacities the planner asks the device for (``cudaOccupancyMaxActiveClusters``) are a parameter; ``H100_CAPACITY``
records them for the packed cluster kernels on an H100 (132 SMs), and the GPU tests check the record.
"""
from __future__ import annotations

from typing import NamedTuple

import numpy as np

SMS = 132          # the H100's SM count
SLOTS = 512        # the reference's FPS block: tie-break (k mod 512, k)
SCRATCH_T = 1024   # threads of fps_global_kernel
SCRATCH_GRID = 32  # its most CTAs; CTA c serves clouds c, c + 32, ...
CTA_SMEM_MAX = 200 * 1024

# X(P, T, packed): fps_cta_kernel<P, T, 0>, and <P, T, 1> where packed
CTA_KERNELS = [(1, 128, 0), (2, 128, 0), (4, 128, 0), (8, 128, 1), (16, 128, 1), (32, 128, 1),
               (1, 256, 0), (2, 256, 0), (4, 256, 0), (8, 256, 1), (16, 256, 1), (32, 256, 1),
               (1, 512, 0), (2, 512, 0), (4, 512, 0), (8, 512, 1), (16, 512, 1),
               (1, 1024, 0), (2, 1024, 0), (4, 1024, 0), (8, 1024, 1)]
# X(P, T, PR, packed): fps_cluster_kernel<P, T, PR, 0>, and <P, T, PR, 1> where packed
CLUSTER_KERNELS = [(4, 128, 4, 1), (8, 128, 8, 1), (16, 128, 16, 1), (32, 128, 32, 1),
                   (2, 256, 2, 0), (4, 256, 4, 1), (8, 256, 8, 1), (16, 256, 16, 1), (32, 256, 32, 1),
                   (1, 512, 1, 0), (2, 512, 2, 0), (4, 512, 4, 1), (8, 512, 8, 1), (16, 512, 16, 1), (32, 512, 16, 1),
                   (2, 1024, 2, 0), (4, 1024, 4, 1), (8, 1024, 8, 1)]
# X(P, PR): fps_cluster_big_kernel<P, 512, PR, 0> and <P, 512, PR, 1>
BIG_KERNELS = [(44, 16), (48, 12), (52, 16)]


class Inst(NamedTuple):
    family: str  # "cta", "cluster", "big" or "scratch"
    P: int       # points per thread (0 for the scratch kernel)
    T: int       # threads per CTA
    PR: int      # points per thread with register-resident coordinates (cluster kernels; P for the others)
    V: int       # 1: the packed chain / update, 0: the plain one

    @property
    def name(self):
        return f"{self.family}_P{self.P}_T{self.T}_PR{self.PR}_V{self.V}"


def _instances():
    out = []
    for P, T, pk in CTA_KERNELS:
        out += [Inst("cta", P, T, P, v) for v in ((0, 1) if pk else (0,))]
    for P, T, PR, pk in CLUSTER_KERNELS:
        out += [Inst("cluster", P, T, PR, v) for v in ((0, 1) if pk else (0,))]
    for P, PR in BIG_KERNELS:
        out += [Inst("big", P, 512, PR, v) for v in (0, 1)]
    return out + [Inst("scratch", 0, SCRATCH_T, 0, 0)]


INSTANCES = _instances()

# clusters of each packed cluster kernel an H100 keeps resident at once: pn2_fps_cluster_capacity(threads, ppt, C) for
# every plan plan_fps can ask about, as read on an H100 80GB HBM3 (132 SMs) with CUDA 12.9
H100_CAPACITY = {
    (128, 8, 16): 58, (128, 16, 8): 62, (128, 16, 16): 28, (128, 32, 4): 62, (128, 32, 8): 30,
    (128, 32, 16): 14, (256, 32, 2): 66, (256, 32, 4): 30, (256, 32, 8): 15, (256, 32, 16): 7,
    (512, 32, 2): 66, (512, 32, 4): 30, (512, 32, 8): 15, (512, 32, 16): 7, (512, 44, 2): 66,
    (512, 44, 3): 39, (512, 44, 4): 30, (512, 44, 5): 22, (512, 44, 6): 17, (512, 44, 7): 15,
    (512, 44, 8): 15, (512, 44, 9): 9, (512, 44, 10): 7, (512, 44, 11): 7, (512, 44, 12): 7,
    (512, 44, 13): 7, (512, 44, 14): 7, (512, 44, 15): 7, (512, 44, 16): 7, (512, 48, 2): 66,
    (512, 48, 3): 39, (512, 48, 4): 30, (512, 48, 5): 22, (512, 48, 6): 17, (512, 48, 7): 15,
    (512, 48, 8): 15, (512, 48, 9): 9, (512, 48, 10): 7, (512, 48, 11): 7, (512, 48, 12): 7,
    (512, 48, 13): 7, (512, 48, 14): 7, (512, 48, 15): 7, (512, 48, 16): 7, (512, 52, 2): 66,
    (512, 52, 3): 39, (512, 52, 4): 30, (512, 52, 5): 22, (512, 52, 6): 17, (512, 52, 7): 15,
    (512, 52, 8): 15, (512, 52, 9): 9, (512, 52, 10): 7, (512, 52, 11): 7, (512, 52, 12): 7,
    (512, 52, 13): 7, (512, 52, 14): 7, (512, 52, 15): 7, (512, 52, 16): 7,
}


def h100_capacity(threads, ppt, cluster, packed=1):
    return H100_CAPACITY.get((threads, ppt, cluster), 0) if packed else 0


class Plan(NamedTuple):
    threads: int
    ppt: int
    cluster: int  # 0: global scratch; 1: single CTA; >= 2: a cluster of that many CTAs (< 1 also runs the scratch)
    pr: int
    packed: int


def pow2_floor(v):
    p = 1
    while p * 2 <= v:
        p *= 2
    return p


def decode_override(threads, ppt, cluster, packed=1, packed_cluster=1):
    """pack_cfg then the override branch of plan_fps: the plan an override names (None: no override)"""
    if threads <= 0:
        return None
    ppt &= 0xFFFFF
    chain = threads & 3
    builtin = packed_cluster if cluster >= 2 else packed
    pk = 1 if chain == 1 else (0 if chain == 2 else builtin)
    threads &= ~3
    pr = 16 if (ppt >= 32 and threads >= 512) else ppt
    if cluster in (-1, -2):  # single CTA with the chain named explicitly
        pk = 1 if cluster == -2 else 0
        cluster = 1
    return Plan(threads, ppt, cluster, pr, pk)


def plan_fps(b, n, sms=SMS, capacity=None, override=None, packed=1, packed_cluster=1):
    """plan_fps(b, n): ``capacity(threads, ppt, cluster, packed)`` as fps_cluster_capacity (0 = unknown, the answer
    without a device); ``override`` the (threads, ppt, cluster) of pn2_set_fps_config or None"""
    capacity = capacity or (lambda t, p, c, k: 0)
    if override is not None:
        ov = decode_override(*override, packed=packed, packed_cluster=packed_cluster)
        if ov is not None:
            return ov
    for limit, t, p in ((128, 128, 1), (256, 128, 2), (512, 256, 2), (1024, 128, 8), (2048, 128, 16), (4096, 256, 16),
                        (8192, 256, 32)):
        if n <= limit:
            return Plan(t, p, 1, p, packed)
    cmax = pow2_floor(sms // (sms if b > sms else b))
    cmax = min(max(cmax, 2), 16)

    def pick(per, C):
        t = 128 if C >= 4 else 256
        pp = 4 if t == 128 else 2
        while pp <= 32:
            if per <= t * pp:
                return Plan(t, pp, C, pp, packed_cluster)
            pp *= 2
        if per <= 256 * 32:
            return Plan(256, 32, C, 32, packed_cluster)
        if per <= 512 * 32:
            return Plan(512, 32, C, 16, packed_cluster)
        return None

    first = None
    C = cmax
    while C >= 2:
        per = (n + C - 1) // C
        if per <= 1024 and C > 2:
            C //= 2
            continue
        p = pick(per, C)
        if p is None:
            break
        first = first or p
        cap = capacity(p.threads, p.ppt, p.cluster, p.packed)
        if cap == 0 or cap >= b:
            return p
        C //= 2
    best, best_cost = None, 1e30

    def consider(p):
        nonlocal best, best_cost
        cap = capacity(p.threads, p.ppt, p.cluster, p.packed)
        waves = (b + cap - 1) // cap if cap > 0 else 1
        cost = waves * (0.3 + 0.07e-3 * p.threads * p.ppt)
        if cap > 0 and cap * p.cluster > sms:
            cost *= 1.3
        if cost < best_cost:
            best, best_cost = p, cost

    if first is not None:
        consider(first)
    widest = pick((n + 15) // 16, 16)
    if widest is not None:
        consider(widest)
    for C in range(16, 1, -1):
        per = (n + C - 1) // C
        if per > 512 * 52:
            break
        consider(Plan(512, 44 if per <= 512 * 44 else (48 if per <= 512 * 48 else 52), C, 16, packed_cluster))
    if best is not None:
        return best
    return Plan(1024, 0, 0, 0, 0)


def dispatch(plan, n, have_temp=True):
    """(instantiation, None) for the kernel fps_dispatch launches for ``plan`` on clouds of stride n, or (None, reason)
    when it refuses the plan"""
    if plan.cluster >= 1 and plan.threads * plan.ppt * plan.cluster < n:
        return None, "capacity"
    if plan.cluster == 1:
        for P, T, pk in CTA_KERNELS:
            if plan.ppt == P and plan.threads == T:
                if 3 * n * 4 > CTA_SMEM_MAX:
                    return None, "smem"
                return Inst("cta", P, T, P, 1 if (pk and plan.packed) else 0), None
        return None, "no_instance"
    C = plan.cluster
    if C >= 2 and plan.ppt > 32:
        if C > 16:
            return None, "cluster_over_16"
        if plan.threads != 512:
            return None, "no_instance"
        for P, PR in BIG_KERNELS:
            if plan.ppt == P:
                return Inst("big", P, 512, PR, 1 if plan.packed else 0), None
        return None, "no_instance"
    if C >= 2:
        if C > 16:
            return None, "cluster_over_16"
        if C & (C - 1):
            return None, "cluster_not_pow2"
        if (C * plan.threads) % SLOTS:
            return None, "ct_not_512"
        for P, T, PR, pk in CLUSTER_KERNELS:
            if plan.ppt == P and plan.threads == T and plan.pr == PR:
                return Inst("cluster", P, T, PR, 1 if (pk and plan.packed) else 0), None
        return None, "no_instance"
    if not have_temp:
        return None, "no_scratch"
    return INSTANCES[-1], None


def capacity_of(inst, C=1):
    """points per cloud an instantiation holds (C: its cluster size); the scratch kernel holds any"""
    if inst.family == "scratch":
        return 1 << 62
    return inst.P * inst.T * (C if inst.family in ("cluster", "big") else 1)


# ------------------------------------------------------------------------------------------------ layouts
class ScanOrder(NamedTuple):
    D: int   # distinct reference slots of one thread's points
    DD: int  # ... that a thread with P points sees
    Q: int   # points per slot residue
    GS: int  # scan-order neighbours per search group of the packed chain


def scan_order(P, T):
    D = 1 if T >= SLOTS else SLOTS // T
    DD = min(D, P)
    Q = P // DD
    return ScanOrder(D, DD, Q, 4 if Q >= 4 else Q)


def owner(inst, k, C=1):
    """Where ``inst`` keeps points k (an int array): dict of arrays rank (CTA in the cluster), thread, warp, j (the
    thread's j-th point), and the in-thread position of the point in its chain: residue (reference slot residue,
    single CTA), group (search group of the packed chains; groups of four in value_argmax_first), streamed (cluster
    kernels: coordinates streamed from shared memory, j >= PR)."""
    k = np.asarray(k, np.int64)
    zero = np.zeros_like(k)
    if inst.family == "scratch":
        t = k % SCRATCH_T
        return dict(rank=zero, thread=t, warp=t // 32, j=k // SCRATCH_T, residue=zero, group=zero, streamed=zero)
    T = inst.T
    t = k % T
    if inst.family == "cta":
        so = scan_order(inst.P, T)
        j = k // T
        e = (j % so.DD) * so.Q + j // so.DD  # scan position: ScanOrder::j_of(e) == j
        return dict(rank=zero, thread=t, warp=t // 32, j=j, residue=j % so.DD, group=e // so.GS, streamed=zero)
    q = k // T
    j = q // C
    return dict(rank=q % C, thread=t, warp=t // 32, j=j, residue=zero, group=j // 4,
                streamed=(j >= inst.PR).astype(np.int64))


# the stages a tie can be decided in, per family and chain
STAGES = {
    "cta_V0": {"scan", "residue", "warp", "cross_warp"},
    "cta_V1": {"group", "group_other", "residue", "warp", "cross_warp"},
    "cluster_V0": {"scan", "reg_stream", "warp", "cross_warp", "cluster"},
    "cluster_V1": {"group", "group_other", "reg_stream", "warp", "cross_warp", "cluster"},
    "big_V0": {"scan", "reg_stream", "warp", "cross_warp", "cluster"},
    "big_V1": {"group", "group_other", "reg_stream", "warp", "cross_warp", "cluster"},
    "scratch_V0": {"scan", "warp", "cross_warp"},
}


def family_key(inst):
    return f"{inst.family}_V{inst.V}"


def stages(inst, winner, others, C=1):
    """For the winner of a step and the other points tied with it (int array; ``winner`` a scalar or one winner per
    entry), the stage of ``inst`` that decides between the winner and each of them (a list of names):

    - ``group`` / ``group_other``: the packed chains' search groups (single CTA) or groups of four
      (value_argmax_first): the same group, or another group of the same thread;
    - ``scan``: the plain chains' in-thread strict '>' scan (same slot residue);
    - ``residue``: the single-CTA scan across slot residues (DD > 1);
    - ``reg_stream``: a register-resident point against a streamed one, in one thread of a cluster kernel;
    - ``warp`` / ``cross_warp``: the warp reduction, the reduction over the CTA's warps;
    - ``cluster``: the exchange between the CTAs of a cluster."""
    others = np.asarray(others, np.int64)
    if not len(others):
        return []
    w = owner(inst, np.broadcast_to(np.asarray(winner, np.int64), others.shape), C)
    o = owner(inst, others, C)
    same_rank = w["rank"] == o["rank"]
    same_thread = same_rank & (w["thread"] == o["thread"])
    same_warp = same_rank & (w["warp"] == o["warp"])
    if inst.V == 1:
        in_thread = np.where(w["group"] == o["group"], "group", "group_other")
        if inst.family == "cta":
            in_thread = np.where((w["group"] != o["group"]) & (w["residue"] != o["residue"]), "residue", in_thread)
    else:
        in_thread = np.where(w["residue"] != o["residue"], "residue", "scan")
    in_thread = np.where(w["streamed"] != o["streamed"], "reg_stream", in_thread)
    out = np.where(same_thread, in_thread, np.where(same_warp, "warp", np.where(same_rank, "cross_warp", "cluster")))
    return [str(s) for s in out]
