"""The engine's own backup (k_backup -> backup_game, launched as b200_run_sims launches it, through b200_debug_backup) and the scalar twins
against the reference's own core.cpp on the designed edge trees of tests/golden/backup_edges_golden.npz: traces across the 32-level
windows up to 512 levels, repeated observations in and across windows, every kind of leaf child list, NaN / inf / huge / subnormal
evaluator outputs and visit counts up to millions.  visit, value and variance must match bit for bit (any NaN equal to any NaN).
With the path cache on the statistics must not change, the returned pc_len must stay at or below the first level that holds an
out-of-date copy under DESIGN §4b's rules, and every level below it must read exactly what the arena holds.
Also the walk's z(n) beyond the host table (n >= 65536, evaluated on the device) against the host libm."""
import os

import numpy as np
import pytest

import backup_edges as BE
import gpu_twins as G

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "backup_edges_golden.npz")
FORMS = {"lp": dict(mode="lp", lp_end_from_obs=False, lp_var_gamma2=True), "lpcpp": dict(mode="lp", lp_end_from_obs=True, lp_var_gamma2=False),
         "single": dict(mode="single"), "vanilla": dict(mode="vanilla")}
F32 = np.float32


@pytest.fixture(scope="module")
def cases():
    cs = BE.load(GOLD)
    assert all(c["digest_ok"] for c in cs), "design() no longer makes the golden's inputs: regenerate tests/golden/backup_edges_golden.npz"
    return cs


@pytest.fixture(scope="module")
def engine(gpu_lib):
    """One-game engines, one per (mode, gamma, path cache), made on first use."""
    from tetris_mcts_b200.engine import BatchedEngine
    made = {}

    def get(mode, gamma, cache=False):
        key = (mode, gamma, cache)
        if key not in made:
            made[key] = BatchedEngine(1, max_nodes=2048, eval_kind="synthetic", gamma=gamma, trace_max=512, path_cache=cache, **FORMS[mode])
        return made[key]
    yield get
    for e in made.values():
        e.close()


def _mismatches(got, want):
    return [name for name, g, w in zip(("visit", "value", "variance"), got, want) if not BE.same_bits(g, w)]


def test_k_backup_matches_reference(engine, cases):
    bad = []
    for i, c in enumerate(cases):
        got, _ = G.debug_backup(engine(c["mode"], c["gamma"]), c)
        m = _mismatches(got, c["out"])
        if m:
            bad.append((i, c["mode"], len(c["trace"]), c["tags"], m))
    assert not bad, bad


def test_scalar_twins_match_reference(gpu_lib, cases):
    bad = []
    for i, c in enumerate(cases):
        m = _mismatches(BE.run(c, G), c["out"])
        if m:
            bad.append((i, c["mode"], len(c["trace"]), c["tags"], m))
    assert not bad, bad


def _f(i32):
    return np.asarray(i32, np.int32).view(np.float32)


def _rule_bound(c, pc, pcl):
    """DESIGN §4b restated: after a backup, entry L holds an out-of-date copy when a child slot it serves from the entry (a first
    occurrence other than the picked one) holds an observation of the trace, or when the own record it reads (its own, level L, or its
    picked child's, level L + 1) belongs to an observation that occurs again higher up the trace (the deeper record holds an intermediate
    value).  Returns the shallowest such level (pcl if none)."""
    o = c["n2o"][c["trace"]]
    D, T = len(o), set(o.tolist())
    first = {}
    for d, x in enumerate(o.tolist()):
        first.setdefault(x, d)
    repeated = [first[x] < d for d, x in enumerate(o.tolist())]
    for L in range(pcl):
        sib = pc["sib"][L]
        if any(sib[a] != 0 and a != sib[7] and int(sib[a]) in T for a in range(7)):
            return L
        if repeated[L] or (L + 1 < D and repeated[L + 1]):
            return L
    return pcl


def _first_incoherent(c, stats, pc, pcl):
    """The shallowest level in [0, pcl) at which a cached value differs from what the arena holds now: the own records of the level and of
    the next, and {val, visit, root} of every slot served from the entry, recomputed as select_trace computes them (clt_val, clt_root)."""
    visit, value, var = stats
    o = c["n2o"][c["trace"]]
    D = len(o)

    def own_ok(d):
        r, x = pc["own"][d], o[d]
        return r[0] == visit[x] and BE.same_bits(_f(r[1]), value[x]) and BE.same_bits(_f(r[2]), var[x])
    for L in range(pcl):
        if not own_ok(L) or (L + 1 < D and not own_ok(L + 1)):
            return L
        sib, s_idx = pc["sib"][L], _f(pc["ent"][L, 7, 1])
        for a in range(7):
            x = int(sib[a])
            if x == 0 or a == sib[7]:
                continue
            e = pc["ent"][L, a]
            with np.errstate(all="ignore"):
                val = (F32(value[x]) + _f(pc["var"][L, a])) - s_idx
                root = np.sqrt(F32(var[x]) / F32(visit[x]))
            if e[2] != visit[x] or not BE.same_bits(_f(e[1]), val) or not BE.same_bits(_f(e[3]), root):
                return L
    return pcl


def test_path_cache_backup(engine, cases):
    n, conservative, truncated, bad = 0, 0, 0, []
    for i, c in enumerate(cases):
        if c["mode"] not in ("lp", "lpcpp"):
            continue
        D = len(c["trace"])
        pcl = D - 1 if c["kind"] == 1 else D
        off, _ = G.debug_backup(engine(c["mode"], c["gamma"], False), c)
        on, pc = G.debug_backup(engine(c["mode"], c["gamma"], True), c, pcl)
        if _mismatches(on, off) or _mismatches(on, c["out"]):
            bad.append((i, "statistics", _mismatches(on, off)))
            continue
        got = int(pc["pc_len"][0])
        rule, true = _rule_bound(c, pc, pcl), _first_incoherent(c, on, pc, pcl)
        if got > rule or got > true:
            bad.append((i, c["tags"], D, "pc_len %d, rule bound %d, first incoherent level %d" % (got, rule, true)))
        n += 1
        truncated += got < pcl
        conservative += got < true
    print("\npath cache: %d LP cases, pc_len truncated in %d, shorter than necessary in %d (%.1f %%)"
          % (n, truncated, conservative, 100.0 * conservative / max(n, 1)))
    assert not bad, bad
    assert truncated > 0


def test_ztab_matches_host_libm(gpu_lib, oracle):
    """z(n) of the walk for every n < 2^24 and 10^6 random n up to 2^31 - 1 against (float) of the host libm's special.h:26-33: the
    table covers n < 65536; beyond it the device evaluates the formula with its own log."""
    rng = np.random.default_rng(7)
    chunks = [np.arange(s, s + (1 << 22), dtype=np.int32) for s in range(0, 1 << 24, 1 << 22)]
    chunks.append(rng.integers(1 << 24, (1 << 31) - 1, 1_000_000, dtype=np.int64).astype(np.int32))
    bad = []
    for n in chunks:
        dev, host = G.ztab(n), oracle.norm_quantile_f32(n)
        diff = ~((dev.view(np.int32) == host.view(np.int32)) | (np.isnan(dev) & np.isnan(host)))
        bad += [(int(k), float(dev[j]), float(host[j])) for j, k in zip(np.nonzero(diff)[0], n[diff])]
    assert not bad, (len(bad), bad[:20])
