"""Bin passes with dead-warp patterns built on purpose, and the model of what bin retirement marks (TEST
INFRASTRUCTURE; tests/test_bin_chain_cases_cpu.py checks it with the C oracle, tests/test_gpu_bin_retirement.py runs
it on the GPU).

A bin pass with rank tables treats a bin as dead once it holds a pod and its remaining amount S[d] is below the call's
smallest request of dimension d in some d.  A resolver warp owns 32 bins of a stage; it is dead when all its bins below
the stage's `n_valid` are, and a stage is retired when all its warps are.  Bins die only by taking a pod, so which warps
and stages are dead when a pass ends follows from the final bins alone: `retirement` below computes it from the
oracle's bins and the launch records, and the library's hook (Engine.last_bin_retirement) must report the same.

How a pattern is built, in the pattern dimension (unit 10):
  - one opener pod per bin, in bin order: 8 leaves 2 (dead: the call's minimum is 3), 7 leaves 3 (live, exactly the
    minimum), 6 leaves 4 (live).  No opener fits a bin already opened, so opener i opens bin i;
  - probe pods of 3 (or 4) then land in the first live bin that has room and kill it;
  - big pods of 9 fit no opened bin: each pushes an entry through every live warp of every patterned stage and opens
    a bin further on.
Column 1 is the pods column (110 per node, 1 per pod); every other column asks 1 of 1000 (never short)."""
import numpy as np

PODS_COL = 1
UNIT_DIM = 10.0
DEAD, LIVE, LIVE4 = 8.0, 7.0, 6.0
PROBE, PROBE4, BIG = 3.0, 4.0, 9.0


def unit_row(D, dim=0):
    u = np.full(D, 1000.0)
    u[dim] = UNIT_DIM
    u[PODS_COL] = 110.0
    return u


def rows(col, D, dim=0):
    """request rows whose pattern dimension is `col` (pods column 1, every other column 1)"""
    col = np.asarray(col, np.float64)
    r = np.ones((len(col), D))
    r[:, dim] = col
    return r


def stage_openers(bits, Tn, live=LIVE):
    """openers of one stage of Tn bins: warp w is live when bit w of `bits` is set (Tn < 32: one warp)"""
    out = []
    for n in range(Tn):
        out.append(live if (bits >> (n // 32)) & 1 else DEAD)
    return out


def tail(n_probe, n_big, every=4, probe=PROBE):
    """probes interleaved with big pods (one big after every `every` probes), then the rest of the bigs"""
    out, b = [], 0
    for i in range(n_probe):
        out.append(probe)
        if (i + 1) % every == 0 and b < n_big:
            out.append(BIG)
            b += 1
    return out + [BIG] * (n_big - b)


def remaining(req, bin_of, unit):
    """[opened bins, D]: each bin's remaining amounts after the pass, subtracted in pod order as the reference does"""
    nb = int(bin_of.max()) + 1 if len(bin_of) and bin_of.max() >= 0 else 0
    S = np.tile(np.asarray(unit, np.float64), (nb, 1))
    for i in np.nonzero(bin_of >= 0)[0]:
        S[bin_of[i]] = S[bin_of[i]] - req[i]
    return S


def minreq(req):
    """the smallest value of every column over every request row of the call (-0.0 folded into +0.0)"""
    return req.min(axis=0) + 0.0


def stage_dead_mask(S, minreq_, lo, Tn, n_valid=None):
    """bit w: warp w of the stage over bins [lo, lo + Tn) is dead (every bin below n_valid is opened and short)"""
    n_valid = Tn if n_valid is None else n_valid
    short = (S < minreq_).any(axis=1) if len(S) else np.zeros(0, bool)
    mask = 0
    for w in range((n_valid + 31) // 32):
        b = np.arange(lo + 32 * w, lo + min(32 * w + 32, n_valid))
        if b[-1] < len(S) and short[b].all():
            mask |= 1 << w
    return mask


def retirement(records, S_by_pool, minreq_, rank=0):
    """(dead warps, retired stages) of the bin passes in `records` (Engine.last_launches of one rank), from each pool's
    final bins (S_by_pool: visiting index -> remaining amounts of its opened bins).  Passes without rank tables (RW = 0)
    or in the streaming form retire nothing.  A record's bin_base is the first bin of the whole pass; in cluster mode
    rank r owns the r-th run of `stages` stages of it.  A bin stage's n_valid is its part of the rank's bin range,
    [bin_base + r * stages * Tn, + stages * Tn): every bin stage is Tn wide, on one GPU and in cluster mode alike."""
    warps = stages = 0
    for r in records:
        if r["pass"] != 1 or r["RW"] == 0 or r["form"] != 0:
            continue
        S = S_by_pool.get(r["pool"], np.zeros((0, len(minreq_))))
        Tn = r["Tn"]
        first = r["bin_base"] + rank * r["stages"] * Tn
        hi = first + r["stages"] * Tn
        for s in range(r["stages"]):
            lo = first + s * Tn
            n_valid = min(Tn, hi - lo)
            m = stage_dead_mask(S, minreq_, lo, Tn, n_valid)
            warps += bin(m).count("1")
            stages += m == (1 << ((n_valid + 31) // 32)) - 1
    return warps, stages


def pool_bins(pack_one, req, acc_pool, units, ignored=None):
    """visiting index -> remaining amounts of the pool's opened bins.  The pods that reached pool t are those no earlier
    pool accounted (acc_pool of the full call is -1 or >= t); pack_one(t, idx) packs rows idx into pool t alone, without
    a size limit, and returns the oracle's bin_of for them: the bins the full call opened in that pool."""
    out = {}
    for t in range(len(units)):
        if ignored is not None and ignored[t]:
            continue
        idx = np.nonzero((acc_pool < 0) | (acc_pool >= t))[0]
        if len(idx):
            out[t] = remaining(req[idx], pack_one(t, idx), units[t])
    return out


# ---------------------------------------------------------------------------------------------------------------------
# named cases: req, unit, knobs, the planned stage width "Tn", and "expect": {stage: dead-warp mask at the end of the
# pass} for the patterned stages (checked on the CPU with the oracle)
# ---------------------------------------------------------------------------------------------------------------------
def _case(openers_by_stage, Tn, tail_, D=2, dim=0, knobs=None):
    col = [v for st in openers_by_stage for v in st] + list(tail_)
    return {"req": rows(col, D, dim), "unit": unit_row(D, dim), "Tn": Tn, "knobs": {"min_stages": 1, **(knobs or {})}}


def _pattern_case(bits_list, Tn=256, n_probe=1, n_big=96, D=2, dim=0, knobs=None):
    """one stage per entry of bits_list; probes eat live bins in order; the expected dead masks follow from which
    live bins the probes reach"""
    n_warps = max(1, (Tn + 31) // 32)
    openers = [stage_openers(b, Tn) for b in bits_list]
    # expected: live bins eaten in bin order by the first n_probe probes
    live_bins = [s * Tn + n for s, st in enumerate(openers) for n, v in enumerate(st) if v == LIVE]
    eaten = set(live_bins[:n_probe])
    expect = {}
    for s, st in enumerate(openers):
        m = 0
        for w in range(n_warps):
            bins = range(s * Tn + 32 * w, s * Tn + min(32 * w + 32, Tn))
            if all(openers[s][b - s * Tn] == DEAD or b in eaten for b in bins):
                m |= 1 << w
        expect[s] = m
    c = _case(openers, Tn, tail(n_probe, n_big), D, dim, knobs)
    c["expect"] = expect
    return c


def _last_live_dies_first():
    """stage 0: warps 0-1 live with 3 left (opener 7), warp 5 live with 4 left (opener 6), the rest dead.  Probes of
    4 fit only warp 5's bins: warp 5, the chain's last live warp, dies in an early tile while warps 0-1 are still live;
    the chain's last warp then moves to warp 1.  Probes of 3 then eat warp 0."""
    Tn = 256
    st = []
    for n in range(Tn):
        w = n // 32
        st.append(LIVE if w in (0, 1) else LIVE4 if w == 5 else DEAD)
    col = st + [PROBE4] * 32 + [BIG] * 300 + [PROBE] * 32 + [BIG] * 300
    c = _case([st], Tn, col[Tn:])
    c["expect"] = {0: 0xFF & ~0x02}
    return c


def _sweep(D=2, dim=0):
    """every non-full pattern of the stage's warps, one per stage (255 at 8 warps, 15 at D = 16's 4 warps), then
    probes that eat the live bins stage by stage (half of them), so every pattern sees traffic"""
    Tn = 128 if D == 16 else 256
    nw = Tn // 32
    pats = list(range((1 << nw) - 1))
    n_live = sum(bin(p).count("1") * 32 for p in pats)
    return _pattern_case(pats, Tn, n_probe=n_live // 2, n_big=64, D=D, dim=dim)


def _widths():
    """stage widths from the narrowest the default plan makes (few pods, min_stages = the GPU's SMs) up to 256"""
    out = {}
    for Tn, ms in ((8, 132), (16, 66), (32, 33), (64, 17), (128, 9), (256, 1)):
        bits = [0x0, 0x1, 0x0, 0x1, 0x0, 0x0] if Tn <= 32 else [0x0, 0x1, 0x2, 0x0, 0x1, 0x0]
        c = _pattern_case(bits, Tn, n_probe=Tn // 2, n_big=0)
        # enough pods for ms stages of Tn bins so that the plan keeps Tn (bigs fill the rest)
        need = ms * Tn - len(c["req"])
        if need > 0:
            c["req"] = np.concatenate([c["req"], rows([BIG] * need, 2)])
        c["knobs"] = {"min_stages": ms}
        out["width_%d" % Tn] = c
    return out


def _retired_then_placing():
    """stages 0-1 all dead after their openers, stage 2 half live: every later tile passes stages 0-1 untouched
    (the retired path must count its pods as forwarded, or `drained` ends the pass early) while stages 2-4 place"""
    return _pattern_case([0x00, 0x00, 0x0F], 256, n_probe=64, n_big=600)


def _min_from_unseen_row(kind):
    """the call's minimum in the pattern dimension is 2, from a row the bin pass never sees (an infeasible pod, or -
    scale_up - a pod a node takes): bins with 2 left are then live, and only warps whose bins hold exactly 0..1 die.
    The case carries an extra row at index 0; the GPU test routes it (infeasible for fulfill_pending)."""
    c = _pattern_case([0x00, 0x0F], 256, n_probe=128, n_big=64)
    extra = rows([2.0], 2)
    if kind == "infeasible":
        extra[0, PODS_COL] = 200.0  # more pods than any node takes
    c["req"] = np.concatenate([extra, c["req"]])
    c["unseen_row"] = kind
    c["expect"] = {0: 0x00, 1: 0x0F}  # 2 left is live now; the probes of 3 fill the 7-bins of stage 1 to 0
    return c


def cases():
    out = {
        "alternating_55": _pattern_case([0x55, 0x55], n_probe=1),
        "alternating_aa": _pattern_case([0xAA, 0xAA], n_probe=1),
        "only_warp0_live": _pattern_case([0x01, 0x01], n_probe=16),
        "only_warp7_live": _pattern_case([0x80, 0x80], n_probe=16),
        "hole_LDL": _pattern_case([0b10101, 0b101], n_probe=40),
        "one_live_in_middle": _pattern_case([0x10, 0x08], n_probe=1),
        "last_live_dies_first": _last_live_dies_first(),
        "sweep_d2": _sweep(2),
        "sweep_d16": _sweep(16),
        "sweep_d8_dim5": _sweep(8, dim=5),
        "retired_then_placing": _retired_then_placing(),
        "min_from_infeasible_row": _min_from_unseen_row("infeasible"),
    }
    out.update(_widths())
    return out


def oracle_pass(oracle_mod, c):
    """the case as one pool without a size limit: the oracle's answer and its bins"""
    req = c["req"]
    o = oracle_mod.fulfill_pending(req, len(req), c["unit"].reshape(1, -1), np.zeros(1, np.int32),
                                   np.array([1 << 30], np.int32), np.zeros(1, np.uint8), 0)
    return o, remaining(req, o["bin_of"], c["unit"])
