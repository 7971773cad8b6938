"""The three floating-point rules a pick turns on, at their rounding boundaries, at every site that evaluates them.

- Imbalance gate (cache_aware.rs:662-670): min and max load over ALL workers; imbalanced ⇔ max − min > abs and
  (max as f32) > (min as f32 · rel), rel an f32.
- Match rate (cache_aware.rs:848-854 for tokens, :917-927 for text): matched as f32 / input as f32 > cache_threshold, 0 input → 0.0;
  the string tree counts chars, not bytes.
- prefix_hash load bound (prefix_hash.rs:116-127): load as f64 ≤ (total + 1) as f64 / n as f64 · load_factor, total over the healthy
  workers; total 0 → every load passes.

Each rule has an exact model here (rationals rounded to a binary format, ties to even), checked against the IEEE arithmetic of numpy
and Python.  The case generators put inputs on each side of each boundary and name the side; some cases are chosen so that a
plausible rewrite of the rule (an algebraically equal form, an unrounded product, a conversion through f64, `>=` for `>`, bytes for
chars) lands on the other side.  The tests without the gpu mark prove every case's side with the exact model and check the oracle
against it.  The gpu tests compare the sites with the oracle on these cases only: fleet_prepare_kernel in event, token-tree and
string-tree mode; host_imbalanced (event mode with a token tree); feedback_resolve_kernel; shard_reduce_kernel on one and two ranks;
tree_select_kernel and string_select_kernel in both batch modes; prefix_fleet_prepare_kernel + prefix_pick_kernel through the host and
the device-batch entry points.  Outputs are filled with a poison value before every call."""
import ctypes as C
import os
import sys
from fractions import Fraction

import numpy as np
import pytest

from oracle import orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PAGE = 16
POISON_IDX = -7
POISON_BRANCH = 0xEE
POISON_U32 = 0xDEADBEEF


# =====================================================================================================================
# exact arithmetic
# =====================================================================================================================
def round_binary(q, bits):
    """The non-negative rational q rounded to the nearest value with a `bits`-bit significand, ties to even.  No exponent range:
    every value here is far from the overflow and subnormal ranges of f32."""
    q = Fraction(q)
    if q == 0:
        return q
    assert q > 0
    n, d = q.numerator, q.denominator
    e = n.bit_length() - d.bit_length()            # 2^e ≤ q < 2^(e+1) after the fix-up
    if (n << max(-e, 0)) < (d << max(e, 0)):
        e -= 1
    scale = Fraction(2) ** (bits - 1 - e)           # q · scale ∈ [2^(bits−1), 2^bits)
    m = q * scale
    i, r = divmod(m.numerator, m.denominator)
    if 2 * r > m.denominator or (2 * r == m.denominator and i & 1):
        i += 1
    return Fraction(i) / scale


def f32(x):
    return round_binary(x, 24)


def f64(x):
    return round_binary(x, 53)


def setting32(v):
    """A Python float handed to an f32 setting (ctypes c_float): the f64 value rounded to f32."""
    return Fraction(float(np.float32(v)))


def f32_next(v, up=True):
    """The f32 neighbour of the positive f32 value v."""
    e = v.numerator.bit_length() - v.denominator.bit_length()
    if (v.numerator << max(-e, 0)) < (v.denominator << max(e, 0)):
        e -= 1
    ulp = Fraction(2) ** (e - 23)
    if not up and v == Fraction(2) ** e:
        ulp /= 2
    return v + ulp if up else v - ulp


# ---- imbalance gate ----
def gate(mn, mx, abs_thr, rel):
    return mx - mn > abs_thr and f32(mx) > f32(f32(mn) * setting32(rel))


GATE_VARIANTS = {   # rewrites the gate must not take
    "via_f64": lambda mn, mx, a, rel: mx - mn > a and f32(f64(mx)) > f32(f32(f64(mn)) * setting32(rel)),   # u64 → f64 → f32
    "unrounded_product": lambda mn, mx, a, rel: mx - mn > a and f32(mx) > f32(mn) * setting32(rel),         # product kept in f64 / FMA
    "ge": lambda mn, mx, a, rel: mx - mn > a and f32(mx) >= f32(f32(mn) * setting32(rel)),
    "abs_ge": lambda mn, mx, a, rel: mx - mn >= a and f32(mx) > f32(f32(mn) * setting32(rel)),
}


# ---- match rate ----
def rate_above(matched, n, thr):
    return n != 0 and f32(f32(matched) / f32(n)) > setting32(thr)


RATE_VARIANTS = {
    "exact": lambda m, n, thr: n != 0 and Fraction(m, n) > setting32(thr),
    "product_f32": lambda m, n, thr: n != 0 and f32(m) > f32(setting32(thr) * f32(n)),   # matched > thr * input, in f32
    "product_f64": lambda m, n, thr: n != 0 and f64(m) > f64(setting32(thr) * f64(n)),   # the same test in f64
}


# ---- prefix_hash load bound ----
def load_ok(load, total, n, factor):
    if total == 0 or n == 0:
        return True
    bound = f64(f64(f64(total + 1) / f64(n)) * Fraction(factor))
    return f64(load) <= bound


BOUND_VARIANTS = {
    "exact": lambda load, t, n, f: t == 0 or n == 0 or load <= Fraction(t + 1, n) * Fraction(f),
    "factor_first": lambda load, t, n, f: t == 0 or n == 0 or f64(load) <= f64(f64(f64(t + 1) * Fraction(f)) / f64(n)),   # (t + 1) * f / c
    "int_division": lambda load, t, n, f: t == 0 or n == 0 or f64(load) <= f64(f64(Fraction(t + 1, n)) * Fraction(f)),  # Python (t + 1) / c
}


# =====================================================================================================================
# gate cases
# =====================================================================================================================
def _int_neighbours(p):
    """(largest integer whose f32 is below p, smallest integer whose f32 is above p) for an integral f32 value p > 0."""
    lo = int(p) - 1
    while f32(lo) >= p:
        lo -= 1
    hi = int(p) + 1
    while f32(hi) <= p:
        hi += 1
    return lo, hi


def gate_cases():
    """[dict(name, mn, mx, abs, rel, open, splits)]: `open` is the side the case names (imbalanced), `splits` the variants of
    GATE_VARIANTS that put it on the other side."""
    cases = []

    def add(name, mn, mx, a, rel, side, splits=()):
        cases.append(dict(name=name, mn=mn, mx=mx, abs=a, rel=rel, open=side == "open", splits=tuple(splits)))

    # the abs part: max − min == abs stays closed, abs + 1 opens (min 0: the f32 part is open for any max > 0)
    for a in (0, 1, 32, 64):
        add(f"abs{a}_diff_eq_min0", 0, a, a, 1.5, "closed", ["abs_ge"] if a else [])
        add(f"abs{a}_diff_above_min0", 0, a + 1, a, 1.5, "open")
    add("abs32_diff_eq_rel0.5", 1000, 1032, 32, 0.5, "closed", ["abs_ge"])
    add("abs32_diff_above_rel0.5", 1000, 1033, 32, 0.5, "open")
    add("rel0_diff_eq", 5, 9, 4, 0.0, "closed", ["abs_ge"])
    add("rel0_diff_above", 5, 10, 4, 0.0, "open")
    # f32(max) == f32(min) * rel exactly → closed; the integers whose f32 is one step below / above
    for mn, rel, a in ((10, 1.5, 4), (1000, 1.1, 50), (2 ** 24, 1.5, 4), (3 * 2 ** 23, 1.6666666, 1), (2 ** 25, 1.1, 4)):
        p = f32(f32(mn) * setting32(rel))
        assert p.denominator == 1, (mn, rel)
        lo, hi = _int_neighbours(p)
        add(f"product_eq_mn{mn}_rel{rel}", mn, int(p), a, rel, "closed", ["ge"])
        add(f"product_below_mn{mn}_rel{rel}", mn, lo, a, rel, "closed")
        add(f"product_above_mn{mn}_rel{rel}", mn, hi, a, rel, "open")
        if f32(int(p) + 1) == p:                       # above 2^24: max + 1 has the same f32 as max
            add(f"product_eq_plus1_mn{mn}_rel{rel}", mn, int(p) + 1, a, rel, "closed", ["ge"])
    # rel not representable in f32
    add("rel1.6666666_3_5", 3, 5, 1, 1.6666666, "closed", ["ge", "unrounded_product"])
    add("rel1.6666667_3_5", 3, 5, 1, 1.6666667, "closed", ["ge"])
    add("rel1.1_7_8", 7, 8, 0, 1.1, "open")
    # the unrounded product disagrees: f32(min · rel) rounds up onto an integral max
    mns = np.concatenate([np.arange(1, 20000), 2 ** 24 + np.arange(20000)]).astype(np.int64)   # above 2^24 every f32 is an integer
    for rel in (1.1, 1.6666666, 1.6666667):
        exact = np.float64(np.float32(mns)) * np.float64(np.float32(rel))    # f32 · f32 is exact in f64
        p = np.float32(exact)
        hit = np.flatnonzero((p == np.floor(p)) & (exact < p) & (p > mns))[:2]
        assert hit.size == 2, rel
        for i in hit:
            add(f"rounded_up_product_mn{int(mns[i])}_rel{rel}", int(mns[i]), int(p[i]), 0, rel, "closed", ["ge", "unrounded_product"])
    # conversions above 2^24 decided by round-half-to-even
    b = 2 ** 24
    add("rne_max_tie_down", b, b + 1, 0, 1.0, "closed")        # b + 1 → b
    add("rne_max_exact", b, b + 2, 0, 1.0, "open")
    add("rne_max_tie_up", b, b + 3, 0, 1.0, "open")            # b + 3 → b + 4
    add("rne_min_tie_up", b + 3, b + 4, 0, 1.0, "closed")      # b + 3 → b + 4
    add("rne_min_tie_down", b + 1, b + 2, 0, 1.0, "open")      # b + 1 → b
    # near 2^60 the direct conversion and the one through f64 disagree: 2^60 + 2^36 + 1 → 2^60 + 2^37 directly, → 2^60 + 2^36 → 2^60
    t = 2 ** 60 + 2 ** 36 + 1
    add("near2^60_max", 2 ** 60, t, 0, 1.0, "open", ["via_f64"])
    add("near2^60_min", t, 2 ** 60 + 2 ** 37, 0, 1.0, "closed", ["via_f64"])
    return cases


GATE_CASES = gate_cases()
GATE_CONFIGS = sorted({(c["abs"], c["rel"]) for c in GATE_CASES})


# =====================================================================================================================
# fleet layouts for the gate: where the min and the max worker sit, and their health
# =====================================================================================================================
LAYOUTS = {   # W → [(min_pos, max_pos, min_flag, max_flag)]; flag: ok | unhealthy | open_circuit
    2: [(0, 1, "ok", "ok"), (1, 0, "ok", "ok")],
    64: [(0, 63, "ok", "ok"), (63, 0, "ok", "ok"), (0, 63, "unhealthy", "ok"), (63, 0, "ok", "open_circuit")],
    65: [(64, 0, "ok", "ok"), (0, 64, "ok", "ok"), (64, 0, "open_circuit", "ok"), (0, 64, "ok", "unhealthy")],
}


def urls_of(n):
    return [f"http://worker-{i}.svc:8000" for i in range(n)]


def layout_fleet(case, W, layout):
    """→ loads, healthy, circuit, hot: every other worker sits between min and max (at max when there is no integer between), and the
    request is cached only on `hot`, a healthy worker that is neither the min nor the max worker (the max worker when W = 2)."""
    min_pos, max_pos, min_flag, max_flag = layout
    mn, mx = case["mn"], case["mx"]
    mid = mn + (mx - mn) // 2 if mx - mn >= 2 else mx
    loads = [mid] * W
    loads[min_pos], loads[max_pos] = mn, mx
    healthy, circuit = [1] * W, [1] * W
    for pos, flag in ((min_pos, min_flag), (max_pos, max_flag)):
        if flag == "unhealthy":
            healthy[pos] = 0
        elif flag == "open_circuit":
            circuit[pos] = 0
    others = [i for i in range(W) if i not in (min_pos, max_pos)]
    hot = others[-1] if others else max_pos
    assert healthy[hot] and circuit[hot]
    return loads, healthy, circuit, hot


def gate_expectation(case, loads, healthy, circuit, hot):
    """(pick, imbalanced) by the closed form: the first healthy argmin when the gate is open, the cached worker otherwise."""
    assert gate(min(loads), max(loads), case["abs"], case["rel"]) == case["open"]
    if not case["open"]:
        return hot, False
    ok = [i for i in range(len(loads)) if healthy[i] and circuit[i]]
    return min(ok, key=lambda i: (loads[i], i)), True


# =====================================================================================================================
# match-rate cases
# =====================================================================================================================
THRESHOLDS = [0.3, 0.5, 0.1, 1 / 3, 0.7, 0.42]   # below 2^14 `matched > thr * input` in f32 agrees with the quotient for the first five: 0.42 splits it


def rate_cases(thr, step):
    """[(name, matched, input, above, splits)] for one threshold; matched is a multiple of `step` (16 for tokens, 1 for chars).  The
    search runs in numpy's IEEE f32 (the exact model is checked against it); the CPU tests prove every case with the exact model."""
    cases, t = [], setting32(thr)
    t32 = np.float32(thr)
    seen = set()

    def add(name, m, n, splits=()):
        if (m, n) not in seen:
            seen.add((m, n))
            cases.append((name, m, n, rate_above(m, n, thr), tuple(splits)))

    m = np.arange(step, (1 << 14) + 1, step, dtype=np.int64)
    cand = [(m, m * t.denominator // t.numerator + d) for d in range(-2, 3)]
    cand = [(a[b >= a], b[b >= a]) for a, b in cand]
    mm = np.concatenate([a for a, _ in cand])
    nn = np.concatenate([b for _, b in cand])
    order = np.lexsort((nn, mm))
    mm, nn = mm[order], nn[order]
    q = np.float32(mm) / np.float32(nn)
    base = q > t32
    # f32(m) / f32(n) == thr exactly: not above; one input token / char either side
    eq = np.flatnonzero(q == t32)
    assert eq.size, thr
    for i in eq[:2]:
        m_, n_ = int(mm[i]), int(nn[i])
        add(f"eq_{m_}/{n_}", m_, n_)
        add(f"above_{m_}/{n_ - 1}", m_, n_ - 1)
        add(f"below_{m_}/{n_ + 1}", m_, n_ + 1)
    variants = {"exact": mm * t.denominator > nn * t.numerator,
                "product_f32": np.float32(mm) > np.float32(t32 * np.float32(nn)),
                "product_f64": np.float64(mm) > np.float64(t32) * np.float64(nn)}
    for v, got in variants.items():
        for i in [i for i in np.flatnonzero(got != base) if (int(mm[i]), int(nn[i])) not in seen][:2]:
            add(f"{v}_disagrees_{int(mm[i])}/{int(nn[i])}", int(mm[i]), int(nn[i]), [v])
    add("zero_input", 0, 0)
    return cases


TOKEN_RATE_CASES = {thr: rate_cases(thr, PAGE) for thr in THRESHOLDS}
TEXT_RATE_CASES = {thr: rate_cases(thr, 1) for thr in THRESHOLDS}
WIDE = {2: "é", 3: "中", 4: "🔥"}


def byte_char_cases(thr):
    """[(name, prefix_chars, prefix_char, tail_chars, tail_char, above)]: texts whose rate over chars and rate over bytes sit on opposite
    sides of thr.  The prefix is what the tree has cached, the tail is new."""
    out = []
    for nb, wide in WIDE.items():
        for prefix_wide in (True, False):
            for m in range(1, 200):
                hit = None
                for n in range(m + 1, 4 * m + 8):
                    tail = n - m
                    pb, tb = (m * nb, tail) if prefix_wide else (m, tail * nb)
                    if rate_above(m, n, thr) != rate_above(pb, pb + tb, thr):
                        hit = n
                        break
                if hit:
                    out.append((f"{nb}byte_{'prefix' if prefix_wide else 'tail'}_{m}/{hit}", m, wide if prefix_wide else "a",
                                hit - m, "b" if prefix_wide else wide, rate_above(m, hit, thr)))
                    break
    return out


BYTE_CHAR_CASES = {thr: byte_char_cases(thr) for thr in THRESHOLDS}


# =====================================================================================================================
# load-bound cases
# =====================================================================================================================
def bound_cases():
    """[dict(name, total, n, factor, load, ok, splits)]: `load` sits on the worker the ring picks, `ok` is the side the case names."""
    cases = []

    def add(name, t, n, f, load, side, splits=()):
        cases.append(dict(name=name, total=t, n=n, factor=f, load=load, ok=side == "ok", splits=tuple(splits)))

    add("bound_exact_5", 11, 3, 1.25, 5, "ok")                 # (11 + 1) / 3 · 1.25 = 5.0
    add("bound_exact_5_plus1", 11, 3, 1.25, 6, "over")
    add("bound_exact_10_n4", 31, 4, 1.25, 10, "ok")
    add("bound_exact_10_n4_plus1", 31, 4, 1.25, 11, "over")
    add("total_zero", 0, 3, 1.25, 0, "ok")
    # two f64 roundings land on the other side of an integer load than the exact rational / (t + 1) · f / c: searched, not picked
    want = {"exact": 3, "factor_first": 3}
    for f in (1.1, 1.2, 1.3, 0.7, 1.15, 0.9, 1.05):
        fa, fb = Fraction(f).numerator, Fraction(f).denominator
        for n in range(2, 40):
            for t in range(n, 3000):
                if not any(want.values()):
                    break
                ref = (float(t + 1) / float(n)) * f
                alt = (float(t + 1) * f) / float(n)
                for load in sorted({int(ref), int(ref) + 1, int(alt), int(alt) + 1}):
                    if not 0 <= load <= t:
                        continue
                    r = load <= ref
                    if want["exact"] and (load * n * fb <= (t + 1) * fa) != r:
                        add(f"vs_exact_t{t}_n{n}_f{f}_load{load}", t, n, f, load, "ok" if r else "over", ["exact"])
                        want["exact"] -= 1
                    elif want["factor_first"] and (load <= alt) != r:
                        add(f"vs_factor_first_t{t}_n{n}_f{f}_load{load}", t, n, f, load, "ok" if r else "over", ["factor_first"])
                        want["factor_first"] -= 1
    assert not any(want.values()), want
    # a total above 2^53: (t + 1) as f64 rounds, so the bound differs from Python's correctly rounded (t + 1) / n
    for t in range(2 ** 53, 2 ** 53 + 64):
        n, f = 3, 1.0
        ref = (float(t + 1) / float(n)) * f
        py = ((t + 1) / n) * f
        if ref != py:
            load = int(max(ref, py))
            add(f"above_2^53_t{t}", t, n, f, load, "ok" if load <= ref else "over", ["int_division"] + (["exact"] if (load <= Fraction(t + 1, n)) != (load <= ref) else []))
            break
    else:
        raise AssertionError("no total above 2^53 separates the two divisions")
    return cases


BOUND_CASES = bound_cases()


def bound_fleet(case, extra_unhealthy=0):
    """→ loads, healthy: worker 0 carries the case's load (the ring's pick is moved onto it by the caller), the other healthy workers
    share the rest of the total; `extra_unhealthy` unhealthy workers with a large load follow (they must not enter the total)."""
    n, t, load = case["n"], case["total"], case["load"]
    rest = t - load
    q, r = divmod(rest, n - 1)
    loads = [load] + [q + (1 if i < r else 0) for i in range(n - 1)] + [10 ** 6] * extra_unhealthy
    healthy = [1] * n + [0] * extra_unhealthy
    assert sum(l for l, h in zip(loads, healthy) if h) == t
    return loads, healthy


# least_ok at the bound: the ring's pick is overloaded and another worker sits exactly on the bound (below 1: factor 0.5)
LEAST_OK_CASES = [   # (name, loads with the ring's pick first, factor, expected index of the walk, first healthy argmin of the ok set)
    ("least_ok_on_bound", [4, 5, 2], 0.5, 2),              # bound (11 + 1) / 3 · 0.5 = 2.0: worker 2 passes
    ("least_ok_one_over", [4, 4, 3], 0.5, 0),              # bound 13 / 3 · 0.5 = 2.1666…: nobody passes → the ring's pick
    ("least_ok_first_of_equal", [9, 2, 2, 2, 9], 0.75, 1),  # bound 25 / 5 · 0.75 = 3.75
]


# =====================================================================================================================
# feedback streams: the gate re-evaluated on running loads
# =====================================================================================================================
def feedback_streams():
    """[dict(name, loads, healthy, hot, abs, rel, n, closes_at)]: closes_at = the first request that sees the gate closed (None: open
    for the whole stream), derived by hand in the comment of each stream and checked against the simulation."""
    b, t60 = 2 ** 24, 2 ** 60
    return [
        # 7 workers at 3 water-fill until max − min = 80 − 16 ≤ 64: 13 rounds of 7 picks
        dict(name="water_fill", loads=[3] * 5 + [80] + [3] * 2, healthy=[1] * 8, hot=7, abs=64, rel=1.5, n=200, closes_at=91),
        # 7 workers tied at the minimum 10, max 20: the f32 part closes at min 14 (20 > 21 is false): 4 rounds of 7 picks
        dict(name="flat_min_ties", loads=[10] * 3 + [20] + [10] * 4, healthy=[1] * 8, hot=7, abs=4, rel=1.5, n=120, closes_at=28),
        # above 2^24 f32(min) moves on every second bump: f32(b + 21) = b + 20, reached by f32(b + 19); exact integers would need b + 21
        dict(name="above_2^24", loads=[b + 21, b, b + 20], healthy=[1] * 3, hot=2, abs=0, rel=1.0, n=64, closes_at=19),
        # an unhealthy worker at 0 pins the global minimum: the gate never closes (without it, min 57 would close it after 42 picks)
        dict(name="unhealthy_pins_min", loads=[50, 50, 0, 50, 50, 50, 120, 50], healthy=[1, 1, 0, 1, 1, 1, 1, 1], hot=7, abs=64, rel=1.5,
             n=300, closes_at=None),
        # near 2^60 the max converts to 2^60 + 2^37 directly and to 2^60 through f64: open for the whole stream
        dict(name="near_2^60", loads=[t60 + 2 ** 36 + 1, t60, t60 + 2 ** 35], healthy=[1] * 3, hot=2, abs=0, rel=1.0, n=64, closes_at=None),
    ]


FEEDBACK_STREAMS = feedback_streams()


def simulate_feedback(s, gate_fn=gate, healthy_only=False):
    """The request stream by the closed form: every request is cached only on `hot`; an open gate sends it to the first healthy argmin,
    a closed one to `hot`; the pick's load is bumped before the next request.  healthy_only: min / max over the healthy workers (the
    mistake the reference does not make).  → (picks, imbalanced flags, final loads)."""
    loads = list(s["loads"])
    picks, imb = [], []
    for _ in range(s["n"]):
        seen = [l for l, h in zip(loads, s["healthy"]) if h or not healthy_only]
        if gate_fn(min(seen), max(seen), s["abs"], s["rel"]):
            p = min((i for i in range(len(loads)) if s["healthy"][i]), key=lambda i: (loads[i], i))
            imb.append(True)
        else:
            p = s["hot"]
            imb.append(False)
        picks.append(p)
        loads[p] += 1
    return picks, imb, loads


# =====================================================================================================================
# CPU: the exact model against IEEE arithmetic, and every case on its named side
# =====================================================================================================================
def test_exact_model_matches_ieee_arithmetic():
    rng = np.random.default_rng(1)
    xs = [0, 1, 2 ** 24 - 1, 2 ** 24 + 1, 2 ** 24 + 3, 2 ** 53 + 1, 2 ** 60 + 2 ** 36 + 1, 2 ** 64 - 1]
    xs += [int(x) >> int(s) for x, s in zip(rng.integers(0, 2 ** 63, size=3000, dtype=np.uint64) * 2 + 1, rng.integers(0, 60, size=3000))]
    for x in xs:
        assert f32(x) == Fraction(float(np.uint64(x).astype(np.float32))), x
        assert f64(x) == Fraction(float(x)), x
    # np.float32(int) goes through f64 and rounds twice: the example the direct conversion must not follow
    x = 2 ** 60 + 2 ** 36 + 1
    assert f32(x) == 2 ** 60 + 2 ** 37 and Fraction(float(np.float32(x))) == 2 ** 60 == f32(f64(x))
    a = rng.integers(1, 2 ** 40, size=2000)
    bb = rng.integers(1, 2 ** 40, size=2000)
    for u, v in zip(a.tolist(), bb.tolist()):
        fu, fv = np.float32(u), np.float32(v)
        assert f32(Fraction(float(fu)) * Fraction(float(fv))) == Fraction(float(fu * fv))
        assert f32(Fraction(float(fu)) / Fraction(float(fv))) == Fraction(float(fu / fv))
        assert f64(Fraction(u) / Fraction(v)) == Fraction(float(u) / float(v))
        assert f64(Fraction(float(u)) * Fraction(1.1)) == Fraction(float(u) * 1.1)
    for thr in THRESHOLDS + [1.1, 1.6666666, 1.6666667]:
        assert setting32(thr) == Fraction(float(C.c_float(thr).value))


def test_gate_cases_sit_on_their_named_side():
    for c in GATE_CASES:
        args = (c["mn"], c["mx"], c["abs"], c["rel"])
        assert c["mn"] <= c["mx"]
        assert gate(*args) == c["open"], c["name"]
        for v in c["splits"]:
            assert GATE_VARIANTS[v](*args) != c["open"], (c["name"], v)
    split = {v for c in GATE_CASES for v in c["splits"]}
    assert split == set(GATE_VARIANTS)
    # the cases the gate has to be pinned on are present
    assert {c["rel"] for c in GATE_CASES} >= {1.1, 1.6666666, 1.6666667, 1.0, 0.5, 0.0}
    assert any(c["mn"] == 0 and c["open"] for c in GATE_CASES) and any(c["mn"] == 0 and not c["open"] for c in GATE_CASES)
    assert any(c["mx"] - c["mn"] == c["abs"] for c in GATE_CASES) and any(c["mx"] - c["mn"] == c["abs"] + 1 and c["open"] for c in GATE_CASES)
    assert any(c["mx"] > 2 ** 24 and f32(c["mx"]) == f32(c["mx"] + 1) for c in GATE_CASES)
    ties = [x for c in GATE_CASES for x in (c["mn"], c["mx"]) if x > 2 ** 24 and x < 2 ** 25 and x % 2 == 1]
    assert any(f32(x) == x - 1 for x in ties) and any(f32(x) == x + 1 for x in ties)   # half-way cases rounded down and up to even
    # equality cases really are equal, and their neighbours one f32 step away
    for c in GATE_CASES:
        if c["name"].startswith("product_"):
            p = f32(f32(c["mn"]) * setting32(c["rel"]))
            kind = c["name"].split("_")[1]
            if kind == "eq":
                assert f32(c["mx"]) == p
            elif kind == "below":
                assert f32(c["mx"]) == f32_next(p, up=False) or p < 2 ** 23
            elif kind == "above":
                assert f32(c["mx"]) == f32_next(p) or p < 2 ** 23


def test_rate_cases_sit_on_their_named_side():
    for cases, step in ((TOKEN_RATE_CASES, PAGE), (TEXT_RATE_CASES, 1)):
        for thr, cs in cases.items():
            t = setting32(thr)
            kinds = set()
            for name, m, n, above, splits in cs:
                assert m % step == 0 and m <= n, name
                assert rate_above(m, n, thr) == above, name
                for v in splits:
                    assert RATE_VARIANTS[v](m, n, thr) != above, (thr, name, v)
                kind = name.split("_")[0]
                kinds.add(kind)
                if kind == "eq":
                    assert f32(f32(m) / f32(n)) == t and not above
                elif kind == "above":
                    assert above
                elif kind == "below":
                    assert not above
            assert {"eq", "above", "below", "zero"} <= kinds, thr
        assert {v for cs in cases.values() for c in cs for v in c[4]} == set(RATE_VARIANTS), step
    for thr, cs in BYTE_CHAR_CASES.items():
        assert {len(c[2].encode()) for c in cs} | {len(c[4].encode()) for c in cs} == {1, 2, 3, 4}, thr
        for name, pm, pc, tn, tc, above in cs:
            text = pc * pm + tc * tn
            assert rate_above(pm, len(text), thr) == above
            assert rate_above(len((pc * pm).encode()), len(text.encode()), thr) != above, (thr, name)


def test_bound_cases_sit_on_their_named_side():
    for c in BOUND_CASES:
        args = (c["load"], c["total"], c["n"], c["factor"])
        assert load_ok(*args) == c["ok"], c["name"]
        for v in c["splits"]:
            assert BOUND_VARIANTS[v](*args) != c["ok"], (c["name"], v)
        # the f64 model equals the IEEE evaluation of the reference's expression
        if c["total"]:
            assert load_ok(*args) == (float(c["load"]) <= (float(c["total"] + 1) / float(c["n"])) * c["factor"])
    assert {v for c in BOUND_CASES for v in c["splits"]} == set(BOUND_VARIANTS)
    assert any(c["total"] + 1 > 2 ** 53 for c in BOUND_CASES) and any(c["total"] == 0 for c in BOUND_CASES)
    assert any(c["ok"] and Fraction(c["total"] + 1, c["n"]) * Fraction(c["factor"]) == c["load"] for c in BOUND_CASES)
    for name, loads, f, want in LEAST_OK_CASES:
        t, n = sum(loads), len(loads)
        assert not load_ok(loads[0], t, n, f), name
        ok = [i for i in range(n) if load_ok(loads[i], t, n, f)]
        assert (min(ok, key=lambda i: (loads[i], i)) if ok else 0) == want, name
    assert Fraction(12, 3) * Fraction(0.5) == 2        # least_ok_on_bound sits exactly on the bound


def test_feedback_streams_close_where_named():
    for s in FEEDBACK_STREAMS:
        picks, imb, _ = simulate_feedback(s)
        closes = next((i for i, x in enumerate(imb) if not x), None)
        assert closes == s["closes_at"], s["name"]
    by = {s["name"]: s for s in FEEDBACK_STREAMS}
    # rounding decides the index: with integer compares the 2^24 stream would close later, and the 2^60 one at once through f64
    exact = lambda mn, mx, a, rel: mx - mn > a and Fraction(mx) > Fraction(mn) * setting32(rel)
    _, imb, _ = simulate_feedback(by["above_2^24"], exact)
    assert imb.index(False) == 22           # the min worker reaches b + 21, then the cached worker at b + 20 is the minimum once
    _, imb, _ = simulate_feedback(by["near_2^60"], GATE_VARIANTS["via_f64"])
    assert imb[0] is False
    # 6 healthy workers at 50 water-fill to 56, where 120 − 56 ≤ 64 would close the gate
    assert simulate_feedback(by["unhealthy_pins_min"], healthy_only=True)[1].index(False) == 36


# ---- the oracle, through its public calls, on every case ----
class OracleSite:
    """An oracle CacheAwarePolicy in one mode ("event": KV-event indexer; "tokens": token tree only; "text": string tree)."""

    def __init__(self, mode, urls, abs_thr, rel, cache_threshold=0.3, reset=True):
        if reset:
            orc.reset_globals()
        self.mode, self.urls = mode, urls
        self.op = orc.CacheAwarePolicy(eviction_interval_secs=0, cache_threshold=cache_threshold, balance_abs_threshold=abs_thr,
                                       balance_rel_threshold=rel, block_size=PAGE)
        self.op.set_workers(urls)
        if mode == "event":
            self.oix = orc.PositionalIndexer(64)
            self.op.attach_indexer("unknown", self.oix)
            self.op.set_block_size("unknown", PAGE)
            self.op.set_kv_event_monitor(True)
            for u in urls:
                self.oix.intern_worker(u)
        self.k = 0

    def fresh_request(self, hot):
        """A request nobody has seen, cached on `hot`: 4 blocks in the index (event) or 4 pages in the token tree, or 24 chars."""
        self.k += 1
        if self.mode == "text":
            req = f"request {self.k:06d} / " + "abcdefghijklm"
            self.op.string_tree().insert_text(req, self.urls[hot])
            return req
        req = np.arange(1000 + 64 * self.k, 1000 + 64 * self.k + 4 * PAGE, dtype=np.uint32)
        if self.mode == "event":
            hs = orc.compute_request_content_hashes(req, PAGE)
            self.blocks = [(10 ** 6 * self.k + i, h) for i, h in enumerate(hs)]
            self.oix.apply_stored(hot, self.blocks)
        else:
            self.op.token_tree().insert_tokens(req, self.urls[hot])
        return req

    def route(self, loads, healthy, circuit, req):
        self.op.set_state(loads, healthy, circuit)
        if self.mode == "text":
            return self.op.select_worker(request_text=req)
        return self.op.select_worker(tokens=req)


WANT_BRANCH = {"event": "event_overlap", "tokens": "tree_match", "text": "tree_match"}


@pytest.mark.parametrize("mode", ["event", "tokens", "text"])
def test_oracle_gate_equals_closed_form(mode):
    for abs_thr, rel in GATE_CONFIGS:
        for W in (2, 65):
            site = OracleSite(mode, urls_of(W), abs_thr, rel)
            for c in (c for c in GATE_CASES if (c["abs"], c["rel"]) == (abs_thr, rel)):
                for layout in LAYOUTS[W]:
                    loads, healthy, circuit, hot = layout_fleet(c, W, layout)
                    want, imb = gate_expectation(c, loads, healthy, circuit, hot)
                    d = site.route(loads, healthy, circuit, site.fresh_request(hot))
                    assert (d.idx, d.branch) == (want, "imbalanced_min_load" if imb else WANT_BRANCH[mode]), (c["name"], layout)


def test_oracle_feedback_equals_closed_form():
    for s in FEEDBACK_STREAMS:
        W = len(s["loads"])
        site = OracleSite("event", urls_of(W), s["abs"], s["rel"])
        req = site.fresh_request(s["hot"])
        site.op.set_state(s["loads"], s["healthy"], [1] * W)
        flat = np.tile(req, s["n"])
        off = np.arange(s["n"] + 1, dtype=np.uint64) * req.size
        idx, br, _, loads = site.op.select_batch_tokens_feedback(flat, off)
        picks, imb, final = simulate_feedback(s)
        assert idx.tolist() == picks, s["name"]
        assert [b == 1 for b in br.tolist()] == imb and all(b in (1, 2) for b in br.tolist()), s["name"]
        assert loads.tolist() == final, s["name"]


def _rate_requests(cases, thr, kind):
    """Token requests: S[:m] + a fresh tail; text requests: T[:m] + a fresh tail.  Every tail is unique, so the closed-form matched
    count of each request is m against any tree built from S (or T) and earlier requests."""
    out = []
    for j, (name, m, n, above, _) in enumerate(cases):
        if kind == "tokens":
            tail = np.arange(2 * 10 ** 6 + 10 ** 5 * j, 2 * 10 ** 6 + 10 ** 5 * j + n - m, dtype=np.uint32)
            out.append((name, np.concatenate([RATE_S[:m], tail]).astype(np.uint32), m, above))
        else:
            tail = "".join(chr(0x5000 + (j * 977 + i) % 20000) for i in range(n - m))
            out.append((name, RATE_T[:m] + tail, m, above))
    return out


RATE_S = np.arange(1, 80000, dtype=np.uint32)                                 # every token distinct: lcp with S is exact
RATE_T = "".join(chr(0x63 + i % 24) if i % 3 else "ñ" for i in range(70000))   # 1- and 2-byte chars that no tail or byte/char case uses


def _text_byte_char_requests(thr):
    return [(name, pc * pm + tc * tn, pc * pm, above) for name, pm, pc, tn, tc, above in BYTE_CHAR_CASES[thr]]


@pytest.mark.parametrize("snapshot", [False, True])
@pytest.mark.parametrize("kind", ["tokens", "text"])
def test_oracle_rate_equals_closed_form(kind, snapshot):
    for thr in THRESHOLDS:
        site = OracleSite(kind, urls_of(4), 64, 1.5, cache_threshold=thr)
        site.op.set_state([0] * 4, [1] * 4, [1] * 4)
        if kind == "tokens":
            site.op.token_tree().insert_tokens(RATE_S[:4096], urls_of(4)[2])
            reqs = _rate_requests(TOKEN_RATE_CASES[thr], thr, kind)
        else:
            site.op.string_tree().insert_text(RATE_T[:4200], urls_of(4)[2])
            reqs = _rate_requests(TEXT_RATE_CASES[thr], thr, kind)
            for name, text, prefix, above in _text_byte_char_requests(thr):
                site.op.string_tree().insert_text(prefix, urls_of(4)[3])
                reqs.append((name, text, len(prefix), above))
        got = _oracle_rate_batch(site.op, [r[1] for r in reqs], kind, snapshot)
        for (name, q, m, above), (_, br, ma, inp) in zip(reqs, got):
            assert ma == m and inp == len(q), (thr, name)
            assert br == ("tree_match" if above else "tree_min_load"), (thr, name)


def _oracle_rate_batch(op, reqs, kind, snapshot):
    """→ [(idx, branch, matched, input)] from the oracle, one request at a time or as one snapshot batch."""
    if snapshot:
        if kind == "tokens":
            flat, off = _flat(reqs)
            idx, br, ma, _ = op.select_batch_tokens(flat, off, snapshot=True)
            return [(int(x), orc.BRANCHES[int(b)], int(m), len(r)) for x, b, m, r in zip(idx, br, ma, reqs)]
        idx, br, ma, inp, _ = op.select_batch_text(reqs, snapshot=True)
        return [(int(x), orc.BRANCHES[int(b)], int(m), int(i)) for x, b, m, i in zip(idx, br, ma, inp)]
    out = []
    for r in reqs:
        d = op.select_worker(tokens=r) if kind == "tokens" else op.select_worker(request_text=r)
        out.append((-1 if d.idx is None else d.idx, d.branch, d.matched, d.input))
    return out


def _flat(reqs):
    flat = np.concatenate([np.asarray(r, np.uint32) for r in reqs]) if sum(len(r) for r in reqs) else np.zeros(0, np.uint32)
    off = np.zeros(len(reqs) + 1, np.uint64)
    np.cumsum([len(r) for r in reqs], out=off[1:])
    return flat, off


REQ = np.arange(5, 5 + 40, dtype=np.uint32)   # the prefix_hash request of every bound case


def ring_pick(urls, healthy):
    opol = orc.PrefixHashPolicy(256, 1.25)
    idx, br = opol.select_worker(urls, [0] * len(urls), healthy, orc.HashRing(urls), REQ)
    assert br == "ring_hit"
    return idx


def bound_scenarios():
    """[(name, factor, urls, loads, healthy, want_idx, want_branch)]: each bound case with the ring's pick carrying the case's load, once
    as is and once with two unhealthy workers of load 10^6 in the slice; then the least_ok cases."""
    out = []
    for c in BOUND_CASES:
        for extra in (0, 2):
            loads, healthy = bound_fleet(c, extra)
            urls = [f"http://b{len(out)}-{i}:8000" for i in range(len(loads))]
            ring = ring_pick(urls, healthy)
            loads[0], loads[ring] = loads[ring], loads[0]                 # the ring's pick carries the case's load
            t, n = c["total"], c["n"]
            if c["ok"]:
                want = (ring, "ring_hit")
            else:
                ok = [i for i in range(len(loads)) if healthy[i] and load_ok(loads[i], t, n, c["factor"])]
                want = (min(ok, key=lambda i: (loads[i], i)) if ok else ring, "load_balance_walk")
            out.append((f"{c['name']}+{extra}unhealthy", c["factor"], urls, loads, healthy) + want)
    for name, ld, f, want in LEAST_OK_CASES:
        urls = [f"http://b{len(out)}-{i}:8000" for i in range(len(ld))]
        healthy = [1] * len(ld)
        ring = ring_pick(urls, healthy)
        order = [ring] + [i for i in range(len(ld)) if i != ring]          # slice position of each entry of `ld`
        loads = [0] * len(ld)
        for k, pos in enumerate(order):
            loads[pos] = ld[k]
        out.append((name, f, urls, loads, healthy, order[want], "load_balance_walk"))
    return out


def test_oracle_bound_equals_closed_form():
    scen = bound_scenarios()
    assert any(h.count(0) for _, _, _, _, h, _, _ in scen)
    flipped = 0
    for name, f, urls, loads, healthy, want, br in scen:
        opol = orc.PrefixHashPolicy(256, f)
        assert opol.select_worker(urls, loads, healthy, orc.HashRing(urls), REQ) == (want, br), name
        if healthy.count(0) and br == "load_balance_walk":
            t_h = sum(l for l, h in zip(loads, healthy) if h)
            flipped += any(load_ok(l, sum(loads), len(loads), f) != load_ok(l, t_h, healthy.count(1), f) for l, h in zip(loads, healthy) if h)
    assert flipped > 0      # counting the unhealthy workers' loads would change a healthy worker's verdict


# =====================================================================================================================
# GPU
# =====================================================================================================================
def _poisoned(n):
    from smg_b200 import _lib
    out = np.full(max(n, 1), POISON_IDX, np.int32)
    info = (_lib.DecisionInfo * max(n, 1))()
    for i in range(max(n, 1)):
        info[i].matched = info[i].input = POISON_U32
        info[i].branch = info[i].nodes = POISON_BRANCH
    return out, info


def _gpu_tokens(pol, ws, reqs):
    """smgx_select_batch_tokens into poisoned outputs → (idx, [(branch, matched, input)])."""
    from smg_b200.policy import _p
    model = pol._push_fleet(ws)
    flat, off = _flat(reqs)
    off = off.astype(np.uint32)
    n = len(reqs)
    out, info = _poisoned(n)
    tok = _p(flat) if flat.size else C.cast(C.create_string_buffer(4), C.c_void_p)
    pol._h.call("smgx_select_batch_tokens", model, tok, _p(off), n, _p(out), C.cast(info, C.c_void_p))
    return out[:n], [(orc.BRANCHES[info[i].branch], info[i].matched, info[i].input) for i in range(n)]


def _gpu_text(pol, ws, texts):
    from smg_b200.policy import TiktokenTokenizer, _p
    model = pol._push_fleet(ws)
    data, off = TiktokenTokenizer._ragged(texts)
    n = len(texts)
    out, info = _poisoned(n)
    pol._h.call("smgx_select_batch_request_text", model, _p(data), _p(off), n, _p(out), C.cast(info, C.c_void_p))
    return out[:n], [(orc.BRANCHES[info[i].branch], info[i].matched, info[i].input) for i in range(n)]


class GpuSite(OracleSite):
    """The same mode on the GPU policy next to the oracle one (workers interned in slice order on both)."""

    def __init__(self, mode, urls, abs_thr, rel, cache_threshold=0.3, tree_batch_mode="sequential"):
        from smg_b200 import BasicWorker, CacheAwareConfig, CacheAwarePolicy
        self.pol = CacheAwarePolicy(CacheAwareConfig(eviction_interval_secs=0, cache_threshold=cache_threshold, balance_abs_threshold=abs_thr,
                                                     balance_rel_threshold=rel, block_size=PAGE), tree_batch_mode=tree_batch_mode)
        self.ws = [BasicWorker(u) for u in urls]
        self.pol.init_workers(self.ws)
        if mode == "event":
            self.mon = self.pol.kv_event_monitor(PAGE)
            self.ix = self.mon.create_indexer("unknown", 64)
            self.pol.set_kv_event_monitor(self.mon)
            for u in urls:
                self.ix.intern_worker(u)
        super().__init__(mode, urls, abs_thr, rel, cache_threshold)   # resets the oracle's clocks after the GPU trees were made

    def fresh_request(self, hot):
        req = super().fresh_request(hot)
        if self.mode == "text":
            self.pol.string_tree().insert_text(req, self.urls[hot])
        elif self.mode == "event":
            self.ix.apply_stored(hot, self.blocks)
        else:
            self.pol.token_tree().insert_tokens(req, self.urls[hot])
        return req

    def set_fleet(self, loads, healthy, circuit):
        for w, l, h, c in zip(self.ws, loads, healthy, circuit):
            w.set_load(int(l)); w.set_healthy(bool(h)); w.set_circuit_ok(bool(c))

    def both(self, loads, healthy, circuit, req):
        """→ (gpu (idx, branch, matched, input), oracle (idx, branch, matched, input)); event-mode overlap scores are in blocks on the GPU."""
        self.set_fleet(loads, healthy, circuit)
        idx, info = _gpu_text(self.pol, self.ws, [req]) if self.mode == "text" else _gpu_tokens(self.pol, self.ws, [req])
        br, ma, inp = info[0]
        if br == "event_overlap":
            ma *= PAGE
        d = self.route(loads, healthy, circuit, req)
        return (int(idx[0]), br, ma, inp), (-1 if d.idx is None else d.idx, d.branch, d.matched, d.input)


# ---- 1. fleet_prepare_kernel, in the three modes ----
@pytest.mark.gpu
@pytest.mark.parametrize("W", [2, 64, 65])
@pytest.mark.parametrize("mode", ["event", "tokens", "text"])
def test_fleet_prepare_gate(mode, W):
    n = 0
    for abs_thr, rel in GATE_CONFIGS:
        site = GpuSite(mode, urls_of(W), abs_thr, rel)
        for c in (c for c in GATE_CASES if (c["abs"], c["rel"]) == (abs_thr, rel)):
            for layout in LAYOUTS[W]:
                loads, healthy, circuit, hot = layout_fleet(c, W, layout)
                want, imb = gate_expectation(c, loads, healthy, circuit, hot)
                got, orc_d = site.both(loads, healthy, circuit, site.fresh_request(hot))
                assert got == orc_d, (c["name"], layout)
                assert got[:2] == (want, "imbalanced_min_load" if imb else WANT_BRANCH[mode]), (c["name"], layout)
                n += 1
        site.pol.close()
    assert n == len(GATE_CASES) * len(LAYOUTS[W])


# ---- 2. host_imbalanced: event mode with a token tree ----
@pytest.mark.gpu
@pytest.mark.parametrize("abs_thr,rel", GATE_CONFIGS)
def test_host_gate_sends_the_batch_down_the_oracle_path(abs_thr, rel):
    """The host's gate picks the path of an event-mode batch (event kernels, or the token tree with its insert); the kernels' gate the
    branch.  Both must agree with the reference on every case, and the tree must hold exactly the oracle's entries afterwards."""
    W = 65
    site = GpuSite("event", urls_of(W), abs_thr, rel)
    cases = [c for c in GATE_CASES if (c["abs"], c["rel"]) == (abs_thr, rel)]
    for c in cases:
        for layout in LAYOUTS[W][:2]:
            loads, healthy, circuit, hot = layout_fleet(c, W, layout)
            got, orc_d = site.both(loads, healthy, circuit, site.fresh_request(hot))
            assert got == orc_d, (c["name"], layout)
            assert site.pol.token_tree().entries() == site.op.token_tree().entries(), (c["name"], layout)
    site.pol.close()


# ---- 3. feedback_resolve_kernel ----
@pytest.mark.gpu
@pytest.mark.parametrize("stream", [s["name"] for s in FEEDBACK_STREAMS])
def test_feedback_gate_on_running_loads(stream):
    from smg_b200.policy import _p
    s = next(x for x in FEEDBACK_STREAMS if x["name"] == stream)
    W = len(s["loads"])
    site = GpuSite("event", urls_of(W), s["abs"], s["rel"])
    site.pol.set_load_feedback(True)
    req = site.fresh_request(s["hot"])
    site.set_fleet(s["loads"], s["healthy"], [1] * W)
    site.op.set_state(s["loads"], s["healthy"], [1] * W)
    flat = np.tile(req, s["n"])
    off = (np.arange(s["n"] + 1, dtype=np.uint64) * req.size)
    model = site.pol._push_fleet(site.ws)
    out, info = _poisoned(s["n"])
    off32 = off.astype(np.uint32)
    site.pol._h.call("smgx_select_batch_tokens", model, _p(flat), _p(off32), s["n"], _p(out), C.cast(info, C.c_void_p))
    oidx, obr, oma, oloads = site.op.select_batch_tokens_feedback(flat, off)
    br = [info[i].branch for i in range(s["n"])]
    assert out.tolist() == oidx.tolist(), [i for i in range(s["n"]) if out[i] != oidx[i]][:5]
    assert br == obr.tolist()
    assert [info[i].matched * PAGE if br[i] == 2 else info[i].matched for i in range(s["n"])] == oma.tolist()
    # the stream the closed form predicts, and the loads it leaves (the library does not keep the bumps: snapshot + picks)
    picks, imb, final = simulate_feedback(s)
    assert out.tolist() == picks and [b == 1 for b in br] == imb
    assert (np.asarray(s["loads"], dtype=object) + np.bincount(out, minlength=W).astype(object)).tolist() == oloads.tolist() == final
    site.pol.close()


# ---- 4. shard_reduce_kernel ----
@pytest.mark.gpu
@pytest.mark.parametrize("abs_thr,rel", GATE_CONFIGS)
def test_shard_reduce_gate_one_rank(abs_thr, rel):
    from smg_b200 import CacheAwareConfig
    from smg_b200.sharding import ShardedEventRouter
    W = 65
    urls = urls_of(W)
    router = ShardedEventRouter(urls, 0, 1, CacheAwareConfig(eviction_interval_secs=0, cache_threshold=0.3, balance_abs_threshold=abs_thr,
                                                             balance_rel_threshold=rel, block_size=PAGE), jump_size=64, max_tokens_per_request=1024)
    site = OracleSite("event", urls, abs_thr, rel)
    for c in (c for c in GATE_CASES if (c["abs"], c["rel"]) == (abs_thr, rel)):
        for layout in LAYOUTS[W]:
            loads, healthy, circuit, hot = layout_fleet(c, W, layout)
            req = site.fresh_request(hot)
            router.indexer.apply_stored(router.local_id(hot), site.blocks)
            router.set_fleet_state(loads, healthy, circuit)
            want, _ = gate_expectation(c, loads, healthy, circuit, hot)
            off = np.array([0, req.size], np.uint32)
            got = router.select(req, off, 1024, lambda a: a)
            d = site.route(loads, healthy, circuit, req)
            assert int(got[0]) == d.idx == want, (c["name"], layout)
    router.policy.close()


TWO_RANK_CONFIGS = [(4, 1.5), (0, 1.0), (1, 1.6666666)]


def _two_rank_worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, ROOT)
    import torch
    import torch.distributed as dist
    from smg_b200 import CacheAwareConfig
    from smg_b200.sharding import ShardedEventRouter
    from tests import test_gpu_pick_thresholds as M
    dist.init_process_group("gloo", rank=rank, world_size=world)
    ndev = torch.cuda.device_count()

    def all_gather(arr):
        t = torch.from_numpy(arr.copy())
        outs = [torch.empty_like(t) for _ in range(world)]
        dist.all_gather(outs, t)
        return np.concatenate([o.numpy() for o in outs])

    W = 130                                       # 65 workers per shard: the min or max at index 64 is past shard 0's first word
    urls = M.urls_of(W)
    fails, n = [], 0
    for abs_thr, rel in TWO_RANK_CONFIGS:
        cfg = CacheAwareConfig(eviction_interval_secs=0, cache_threshold=0.3, balance_abs_threshold=abs_thr, balance_rel_threshold=rel,
                               block_size=M.PAGE)
        router = ShardedEventRouter(urls, rank, world, cfg, jump_size=64, device_id=rank % max(ndev, 1), max_tokens_per_request=1024)
        router.connect_peers(all_gather)
        site = M.OracleSite("event", urls, abs_thr, rel)
        for c in (c for c in M.GATE_CASES if (c["abs"], c["rel"]) == (abs_thr, rel)):
            for min_pos, max_pos in ((64, 129), (129, 64), (0, 65), (65, 0)):   # min and max on different shards
                loads, healthy, circuit, hot = M.layout_fleet(c, W, (min_pos, max_pos, "ok", "ok"))
                req = site.fresh_request(hot)
                if router.owns(hot):
                    router.indexer.apply_stored(router.local_id(hot), site.blocks)
                router.set_fleet_state(loads, healthy, circuit)
                off = np.array([0, req.size], np.uint32)
                got = router.select(req, off, 1024, all_gather)
                fused = router.select_fused(req, off, 1024)
                want, _ = M.gate_expectation(c, loads, healthy, circuit, hot)
                d = site.route(loads, healthy, circuit, req)
                if not (int(got[0]) == int(fused[0]) == d.idx == want):
                    fails.append((c["name"], min_pos, int(got[0]), int(fused[0]), d.idx, want))
                n += 1
        router.policy.close()
    ret[rank] = (fails, n)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.gpu
def test_shard_reduce_gate_two_ranks():
    """Two ranks share cuda:0 (gloo all-gather and the peer-memory exchange); each case puts the min on one shard and the max on the
    other, so only the merged min / max opens the gate."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    ret = ctx.Manager().dict()
    procs = [ctx.Process(target=_two_rank_worker, args=(r, 2, 29711, ret)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(600)
    assert all(p.exitcode == 0 for p in procs)
    want_n = 4 * sum(1 for c in GATE_CASES if (c["abs"], c["rel"]) in TWO_RANK_CONFIGS)
    for r in range(2):
        fails, n = ret[r]
        assert not fails and n == want_n, (r, fails[:5])


# ---- 5. the match rate in the tree kernels ----
@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["sequential", "snapshot"])
@pytest.mark.parametrize("kind", ["tokens", "text"])
@pytest.mark.parametrize("thr", THRESHOLDS)
def test_tree_rate_boundary(thr, kind, mode):
    urls = urls_of(4)
    site = GpuSite(kind, urls, 64, 1.5, cache_threshold=thr, tree_batch_mode=mode)
    site.set_fleet([0] * 4, [1] * 4, [1] * 4)
    site.op.set_state([0] * 4, [1] * 4, [1] * 4)
    if kind == "tokens":
        for t in (site.pol.token_tree(), site.op.token_tree()):
            t.insert_tokens(RATE_S[:4096], urls[2])
        reqs = _rate_requests(TOKEN_RATE_CASES[thr], thr, kind)
        reqs.append(("zero_tokens", np.zeros(0, np.uint32), 0, False))
    else:
        for t in (site.pol.string_tree(), site.op.string_tree()):
            t.insert_text(RATE_T[:4200], urls[2])
        reqs = _rate_requests(TEXT_RATE_CASES[thr], thr, kind)
        for name, text, prefix, above in _text_byte_char_requests(thr):
            for t in (site.pol.string_tree(), site.op.string_tree()):
                t.insert_text(prefix, urls[3])
            reqs.append((name, text, len(prefix), above))
        reqs.append(("zero_chars", "", 0, False))
    qs = [r[1] for r in reqs]
    idx, info = _gpu_tokens(site.pol, site.ws, qs) if kind == "tokens" else _gpu_text(site.pol, site.ws, qs)
    want = _oracle_rate_batch(site.op, qs, kind, mode == "snapshot")
    for i, (name, q, m, above) in enumerate(reqs):
        assert (int(idx[i]),) + info[i] == want[i], (name, info[i], want[i])
        assert info[i] == ("tree_match" if above else "tree_min_load", m, len(q)), name
    site.pol.close()


# ---- 6. the prefix_hash load bound ----
@pytest.mark.gpu
def test_prefix_bound_host_and_device_entries():
    from smg_b200 import BasicWorker, PrefixHashConfig, PrefixHashPolicy, _lib
    from smg_b200.policy import PREFIX_BRANCHES, _p
    pols = {}
    for k, (name, f, urls, loads, healthy, want, want_br) in enumerate(bound_scenarios()):
        pol = pols.get(f) or pols.setdefault(f, PrefixHashPolicy(PrefixHashConfig(prefix_token_count=256, load_factor=f)))
        ring = pol.hash_ring(urls, model=f"bound-{k}")
        ws = [BasicWorker(u) for u in urls]
        for w, l, h in zip(ws, loads, healthy):
            w.set_load(int(l)); w.set_healthy(bool(h))
        model = pol._push_fleet(ws, ring)
        off = np.array([0, REQ.size], np.uint32)
        # host-buffer entry
        out, info = _poisoned(1)
        pol._h.call("smgx_prefix_hash_select_batch_tokens", model, _p(REQ), _p(off), 1, None, _p(out), C.cast(info, C.c_void_p))
        assert (int(out[0]), PREFIX_BRANCHES[info[0].branch]) == (want, want_br), name
        # device-batch entry
        h, L = pol._h, pol._h.L
        err = _lib.new_err()
        d_tok = L.smgx_device_alloc(h.p, REQ.nbytes, C.byref(err))
        d_off = L.smgx_device_alloc(h.p, off.nbytes, C.byref(err))
        d_out = L.smgx_device_alloc(h.p, 4, C.byref(err))
        h.call("smgx_memcpy_h2d", d_tok, REQ.ctypes.data_as(C.c_void_p), REQ.nbytes)
        h.call("smgx_memcpy_h2d", d_off, off.ctypes.data_as(C.c_void_p), off.nbytes)
        poison = np.full(1, POISON_IDX, np.int32)
        h.call("smgx_memcpy_h2d", d_out, poison.ctypes.data_as(C.c_void_p), 4)
        vp = C.c_void_p * 1
        h.call("smgx_prefix_hash_select_many_tokens_device", model, 1, vp(d_tok), vp(d_off), (C.c_uint32 * 1)(1), vp(d_out))
        h.call("smgx_synchronize")
        got = np.zeros(1, np.int32)
        h.call("smgx_memcpy_d2h", got.ctypes.data_as(C.c_void_p), d_out, 4)
        for d in (d_tok, d_off, d_out):
            L.smgx_device_free(h.p, d)
        assert int(got[0]) == want, name
        # and the oracle through its batch call
        oidx, obr, _ = orc.PrefixHashPolicy(256, f).select_batch(urls, loads, healthy, orc.HashRing(urls), REQ, off.astype(np.uint64))
        assert (int(oidx[0]), orc.PREFIX_BRANCHES[int(obr[0])]) == (want, want_br), name
