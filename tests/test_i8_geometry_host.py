"""The launch geometry of the tensor-core sweep (fp_sweep_i8.cu), on the host (CPU): a Python mirror of the rules
``build_i8_planes`` and ``launch_i8`` apply, with their constants read from the source, and ``CASES``, the packs
tests/test_gpu_i8_geometry.py sweeps against the longdouble truth. A geometry the rules can produce that no case
covers fails here, naming it; so does a case that covers nothing another case does not.

What is picked at run time, per pulsar or per pack:
  * operand rows ``rows = ceil((m + 1) / 32) * 32`` (the basis rows and the w row C^-1 r), swept in
    ``ceil(rows / 128)`` passes over the TOAs, one per row group; the last group has 32, 64, 96 or 128 rows (consumer
    warpgroup 1 idles when it has 64 or fewer) and holds the w row at ``row == m``;
  * stages ``nst = ceil(n / 32)``: the two producer warpgroups take alternate global stage indices, carried across
    passes and items, so an odd ``nst`` swaps their assignment from one pass or item to the next;
  * the G-ring depth ``gst = min(8, (220 KiB - SMEM_FIXED) / gslot)``, ``gslot = 7 * min(rows_max, 128) * 32``: a
    property of the pack (its widest pulsar), so a narrow pulsar in a pack with a wide one runs on the shallow ring;
  * items per CTA: ``grid = min(P * ceil(F / 16), SMs)``, each CTA sweeping items blockIdx.x, + grid, ...;
    ring positions, parities and the double-buffered producer sums carry over from item to item."""
import os
import re
from collections import namedtuple

SRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "fastfp_b200", "csrc",
                   "fp_sweep_i8.cu")
SMS = 132  # SMs of an H100 SXM: the grid of one launch is min(items, SMs)
MAX_N = 16384  # TOAs per pulsar the int32 accumulators carry exactly (7 products of |digit|^2 <= 2^14 per TOA)


def _source():
    with open(SRC) as fh:
        return fh.read()


def constants():
    """Every ``constexpr int`` of namespace i8 and ``SMEM_FIXED``, evaluated in source order; the G-ring budget and
    depth cap of ``launch_i8``."""
    src = _source()
    env = {}
    for decl in re.findall(r"constexpr int ([^;]+);", src[:src.index("struct Args")]):
        for part in decl.split(","):
            name, expr = (s.strip() for s in part.split("=", 1))
            env[name] = int(eval(expr, {}, dict(env)))
    expr = re.search(r"constexpr size_t SMEM_FIXED\s*=([^;]+);", src).group(1)
    env["SMEM_FIXED"] = int(eval(" ".join(expr.replace("(size_t)", "").split()), {}, dict(env)))
    budget = re.search(r"const size_t budget = ([^;]+) - SMEM_FIXED;", src).group(1)
    env["BUDGET"] = int(eval(budget, {}, {})) - env["SMEM_FIXED"]
    cap = re.search(r"gst = gst > (\d+) \? (\d+) : gst;", src)
    assert cap.group(1) == cap.group(2)
    env["GST_CAP"] = int(cap.group(1))
    return env


C = constants()
GROUP = 128  # operand rows per row group: the two consumer warpgroups' 64 each
assert C["NCONS"] * 64 == GROUP and C["RS"] == 5 * GROUP


def rows(m):
    return -(-(m + 1) // 32) * 32


def groups(m):
    return -(-rows(m) // GROUP)


def last_rows(m):
    return rows(m) - GROUP * (groups(m) - 1)


def nst(n):
    return -(-n // C["KT"])


def gst(rows_max):
    gslot = C["NPL"] * min(rows_max, GROUP) * C["KT"]
    return min(C["GST_CAP"], C["BUDGET"] // gslot)


def items_per_cta(P, F):
    """The most items one CTA sweeps: the round-robin over min(items, SMs) CTAs."""
    nwork = P * -(-F // C["NF"])
    return -(-nwork // min(nwork, SMS))


def takes(m, n, blockn=False):
    """Whether the tensor sweep takes a pulsar (``i8_takes``); a non-finite G or w, or a failed factor, still sends
    it to the fp64 kernel at pack time."""
    return not blockn and m + 1 <= C["RS"] and n <= MAX_N


# ---- the cases -------------------------------------------------------------------------------------------------------
# A pulsar is (n_tm, ncomps, n): m = n_tm + 2 ncomps basis columns (white noise only when ncomps = 0), n TOAs.
# F = 131 is the 131-bin grid of test_sweep_instantiations_host.sweep_freqs (red-noise bins, f <= 0, bins past the
# Cody-Waite range, a tile straddling every pulsar's cold-path threshold, a ragged last tile); a larger F is a plain
# grid of that many bins above the red-noise band, long enough for several items per CTA.
Pack = namedtuple("Pack", "name psrs F")

CASES = [
    # ring of 8: every pulsar has at most 64 operand rows; nst = 1 (one producer group idles the whole pass)
    Pack("ring 8", ((5, 0, 31), (7, 10, 64), (20, 20, 97)), 131),
    # ring of 7: one pulsar of 96 rows sizes the ring for the narrower ones
    Pack("ring 7", ((30, 30, 159), (9, 0, 96), (10, 15, 225)), 131),
    # ring of 5: one or more groups of every size, the w row alone in groups 2-5, odd and even nst
    Pack("ring 5, 1-2 groups", ((67, 30, 160), (12, 10, 257), (40, 30, 191), (38, 30, 128),
                                (8, 60, 193), (41, 60, 193), (73, 60, 224), (99, 60, 287), (130, 60, 255)), 131),
    Pack("ring 5, 3 groups", ((136, 60, 449), (180, 60, 385), (200, 60, 479), (263, 60, 447)), 131),
    Pack("ring 5, 4 groups", ((264, 60, 481), (330, 60, 544), (322, 60, 449), (371, 60, 543)), 131),
    Pack("ring 5, 5 groups", ((392, 60, 641), (480, 60, 607), (455, 60, 609), (519, 60, 704)), 131),
    # two groups of 32 stages (nst = 1 in each pass: the stage assignment flips every pass)
    Pack("nst 1, 2 groups", ((20, 60, 31),), 131),
    # several items per CTA: two pulsars of 224 rows in 2 groups with an odd nst; mixed widths in one group each
    Pack("items 5+, row groups", ((100, 50, 449), (80, 60, 705)), 2 * 16 * 66 * 5 - 5),
    Pack("items 5+, mixed widths", ((12, 0, 321), (10, 30, 512), (40, 30, 287), (7, 60, 1025), (16, 0, 33)),
         16 * 133 - 9),
]

# noise-marginalised packs: the per-draw columns are the last 2 ncomps (rows mfix = n_tm .. m - 1), which leave stage
# A as z' rows; the blocks of the wide ones straddle a row-group boundary
NM_CASES = [
    Pack("nmfp ring 8", ((10, 15, 320),), 40),
    Pack("nmfp ring 7", ((30, 30, 257),), 40),
    Pack("nmfp 2 groups, last 128", ((120, 55, 417),), 40),
    Pack("nmfp 5 groups, last 32", ((400, 60, 609),), 40),
    Pack("nmfp ring 5, 3 groups, last 64 + narrow", ((4, 10, 96), (180, 60, 385)), 40),
]


def psr_geometry(q):
    n_tm, nc, n = q
    m = n_tm + 2 * nc
    return dict(m=m, n=n, rows=rows(m), groups=groups(m), last=last_rows(m), nst=nst(n), mfix=n_tm)


def pack_gst(pack):
    return gst(max(rows(q[0] + 2 * q[1]) for q in pack.psrs))


def label(pack, p):
    """"rows 224, 2 groups, last 96, gst 5, nst 47" (+ m, n)"""
    g = psr_geometry(pack.psrs[p])
    return (f"{pack.name}, pulsar {p}: rows {g['rows']}, {g['groups']} groups, last {g['last']}, gst {pack_gst(pack)}, "
            f"nst {g['nst']} (m = {g['m']}, n = {g['n']})")


def covered(pack):
    """The geometry items one Fp pack covers."""
    out = set()
    G = pack_gst(pack)
    out.add(("ring depth", G))
    ms = set()
    for q in pack.psrs:
        g = psr_geometry(q)
        ms.add(g["rows"])
        out.add(("groups x last-group rows", g["groups"], g["last"]))
        if g["m"] % GROUP == 0:
            out.add(("w row alone in group", g["groups"]))
        if g["nst"] == 1:
            out.add(("nst = 1", "groups >= 2" if g["groups"] >= 2 else "1 group"))
        if g["groups"] >= 2:
            out.add(("nst parity with groups >= 2", g["nst"] % 2))
        out.add(("n mod 32", g["n"] % 32))
        own = gst(g["rows"])
        if own != G:
            out.add(("narrow pulsar on a wider pulsar's ring", own, G))
    if items_per_cta(len(pack.psrs), pack.F) >= 5:
        if any(psr_geometry(q)["groups"] >= 2 for q in pack.psrs):
            out.add(("items per CTA >= 5", "row groups"))
        if len(ms) >= 2:
            out.add(("items per CTA >= 5", "mixed widths"))
    return out


def nm_covered(pack):
    out = {("nmfp ring depth", pack_gst(pack))}
    for q in pack.psrs:
        g = psr_geometry(q)
        out.add(("nmfp last-group rows", g["last"]))
        if g["mfix"] // GROUP != (g["m"] - 1) // GROUP:
            out.add(("nmfp per-draw block straddles a row group", g["groups"]))
    return out


def required():
    """Everything the rules can produce that the Fp cases must cover."""
    req = set()
    all_rows = range(32, C["RS"] + 1, 32)
    depths = sorted({gst(r) for r in all_rows})
    req |= {("ring depth", d) for d in depths}
    req |= {("groups x last-group rows", groups(m), last_rows(m)) for m in range(1, C["RS"])}
    req |= {("w row alone in group", groups(m)) for m in range(GROUP, C["RS"], GROUP)}
    req |= {("nst = 1", "1 group"), ("nst = 1", "groups >= 2")}
    req |= {("nst parity with groups >= 2", k) for k in (0, 1)}
    req |= {("n mod 32", r) for r in (0, 1, C["KT"] - 1)}
    req |= {("narrow pulsar on a wider pulsar's ring", a, b) for a in depths for b in depths if a > b}
    req |= {("items per CTA >= 5", "row groups"), ("items per CTA >= 5", "mixed widths")}
    return req


def nm_required():
    req = {("nmfp ring depth", d) for d in {gst(r) for r in range(32, C["RS"] + 1, 32)}}
    req |= {("nmfp last-group rows", r) for r in (32, 64, 96, 128)}
    req |= {("nmfp per-draw block straddles a row group", g) for g in (2, 3, 5)}
    return req


# ---- tests -----------------------------------------------------------------------------------------------------------

def test_constants_and_the_rules_they_give():
    assert (C["NPL"], C["KT"], C["NF"], C["SST"], C["VST"]) == (7, 32, 16, 8, 8)
    assert C["S_STAGE"] == 7168 and C["V_STAGE"] == 512 and C["SMEM_FIXED"] == 66720
    # the depths the rule gives today: 8 slots up to 64 rows, 7 at 96, 5 at 128 or more
    assert {r: gst(r) for r in (32, 64, 96, 128, 640)} == {32: 8, 64: 8, 96: 7, 128: 5, 640: 5}
    assert all(gst(r) >= 2 for r in range(32, C["RS"] + 1, 32))  # launch_i8 refuses fewer
    assert (rows(127), groups(127), last_rows(127)) == (128, 1, 128)
    assert (rows(128), groups(128), last_rows(128)) == (160, 2, 32)
    assert (rows(639), groups(639), last_rows(639)) == (640, 5, 128)
    assert (nst(1), nst(32), nst(33)) == (1, 1, 2)
    assert items_per_cta(1, 16) == 1 and items_per_cta(2, 16 * 66 + 1) == 2 and items_per_cta(5, 16 * 133) == 6


def test_routing_rule():
    """Diagonal N per pack, m + 1 <= 640 operand rows and n <= 16384 TOAs per pulsar; a pulsar whose G or w is not
    finite, or whose factor failed, stays on the fp64 kernel."""
    src = _source()
    body = re.search(r"static bool i8_takes\([^)]*\) \{\s*return ([^;]+);", src).group(1)
    assert body == f"!pk->ecorr && pm.m + 1 <= i8::RS && pm.n <= {MAX_N}", body
    ok = re.search(r"const bool ok = ([^;]+);", src).group(1)
    assert "bad[p] == 0" in ok and "pk->info[p] == 0" in ok and "i8_nst > 0" in ok, ok
    assert takes(639, MAX_N) and not takes(640, 100) and not takes(10, MAX_N + 1) and not takes(10, 100, blockn=True)
    for pack in CASES + NM_CASES:
        for q in pack.psrs:
            g = psr_geometry(q)
            assert takes(g["m"], g["n"]), pack.name


def test_cases_cover_every_geometry():
    got = set().union(*(covered(p) for p in CASES))
    missing = sorted(required() - got, key=str)
    assert not missing, "geometries no case covers: " + "; ".join(map(str, missing))
    assert got <= required(), sorted(got - required(), key=str)
    nm_got = set().union(*(nm_covered(p) for p in NM_CASES))
    missing = sorted(nm_required() - nm_got, key=str)
    assert not missing, "noise-marginalised geometries no case covers: " + "; ".join(map(str, missing))


def test_every_case_is_needed():
    """Each case covers something no other case does, so deleting one fails test_cases_cover_every_geometry."""
    for cases, cov in ((CASES, covered), (NM_CASES, nm_covered)):
        for i, pack in enumerate(cases):
            rest = set().union(*(cov(p) for j, p in enumerate(cases) if j != i))
            assert cov(pack) - rest, f"{pack.name} covers nothing the other cases do not"


def test_cases_are_well_formed():
    for pack in CASES + NM_CASES:
        names = [p.name for p in CASES + NM_CASES]
        assert names.count(pack.name) == 1
        for q in pack.psrs:
            n_tm, nc, n = q
            assert n_tm >= 1 and n >= n_tm and nc >= 0, pack.name  # the timing basis needs n >= n_tm TOAs
        if pack in NM_CASES:
            assert all(1 <= 2 * q[1] <= 128 for q in pack.psrs), pack.name  # per-draw block of 1..128 columns
    # the w row of the 5-group pulsars: alone (m = 512) and at the very end (m = 639)
    ms = {psr_geometry(q)["m"] for p in CASES for q in p.psrs}
    assert {128, 256, 384, 512, 639, 127} <= ms
