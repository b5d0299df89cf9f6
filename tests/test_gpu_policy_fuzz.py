"""Event-driven policies on the GPU against oracle/policy_oracle.c where the warp kernels change path at a chunk of 32:
the random cases of tests/test_policy_fuzz_cpu.py as the heterogeneous replicas of one handle (warp and thread
kernels, whole runs and resumed windows), and targeted cases for each edge -- bursts of 31 .. 200 arrivals, more
than 32 completions at one event (alone and tied with a burst), pending times whose chunk sum passes 2^31 - 1, and
sjf on 8192 nodes, whose node table needs more than 48 KB of shared memory.  Each targeted test asserts from the
oracle's output that its edge really occurs."""
import numpy as np
import pytest

from test_policy_fuzz_cpu import GPU_SEEDS, INT32_MAX, POLICIES, _event_identity, overflow_case, overflow_policies, policy_case

pytestmark = pytest.mark.gpu


def _run(cases, engine=0, rows_cap=0, max_ticks=0, windows=None):
    """cases: (cluster, policy, table) per replica -> per replica (rows, recs, finish order, stats).  With max_ticks the
    run is resumed launch after launch, each one stopping after max_ticks events or rows_cap rows, whichever comes
    first; `windows` (a list) then receives per replica the rows of every launch after which it was not done yet"""
    from gpuschedule_b200 import capi
    with capi.Engine(device=0, nsims=len(cases)) as eng:
        eng.set_engine(engine)             # 0: warp-cooperative kernels, 2: thread-per-replica fallback
        for i, (cluster, pol, table) in enumerate(cases):
            eng.config(i, cluster, pol)
            eng.load_trace(i, table)
        if max_ticks == 0:
            rows = eng.run_all(rows_cap=rows_cap)
        else:
            parts, seen, launches = [[] for _ in cases], [0] * len(cases), 0
            wins = [[] for _ in cases]
            while True:
                eng.run(max_ticks, rows_cap)
                launches += 1
                pending = 0
                for s in range(len(cases)):
                    st = eng.stats(s)
                    if st.ticks > seen[s]:
                        parts[s].append(eng.fetch_rows(s, seen[s], st.ticks - seen[s]))
                    if not st.done:
                        wins[s].append(st.ticks - seen[s])
                    seen[s] = st.ticks
                    pending += 0 if st.done else 1
                if pending == 0:
                    break
            assert launches > 1
            rows = [np.concatenate(p) for p in parts]
            if windows is not None:
                windows.extend(wins)
        out = []
        for i in range(len(cases)):
            recs, order = eng.fetch_jobs(i)
            out.append((rows[i], recs, order, eng.stats(i)))
        return out


def _assert_same(ref, got, tag):
    rows, recs, order, st = got
    assert st.status == 0 and st.done == 1, tag
    assert st.ticks == ref.ticks, (tag, st.ticks, ref.ticks)
    if rows.tobytes() != ref.rows.tobytes():
        bad = next(i for i in range(min(len(rows), len(ref.rows))) if rows[i].tobytes() != ref.rows[i].tobytes())
        raise AssertionError(f"{tag} row {bad}: {rows[bad]} != {ref.rows[bad]}")
    assert recs.tobytes() == ref.recs.tobytes(), tag
    assert np.array_equal(order, ref.finish_order), tag
    assert st.events == ref.events, (tag, st.events, ref.events)


@pytest.fixture(scope="module")
def fuzz_cases():
    import oracle
    cases = [policy_case(seed) for seed in GPU_SEEDS]
    return cases, [oracle.run_policy(c.cluster, c.policy, c.table) for c in cases]


@pytest.mark.parametrize("engine", [0, 2], ids=["warp", "thread"])
def test_policy_fuzz_matches_oracle(fuzz_cases, engine):
    """240 random clusters / traces / policies (sjf, dlas, dlas-gpu, gittins) as the replicas of ONE handle"""
    cases, refs = fuzz_cases
    got = _run([(c.cluster, c.policy, c.table) for c in cases], engine=engine)
    for c, ref, g in zip(cases, refs, got):
        _assert_same(ref, g, f"seed {c.seed} {c.name} {c.ckw} {c.pkw} n={c.table.n}")
    # the quirk-Q25 completion of a job preempted after it joined an end list is among them
    assert sum(_event_identity(c, r) > 0 for c, r in zip(cases, refs)) >= 5


@pytest.mark.parametrize("engine", [0, 2], ids=["warp", "thread"])
@pytest.mark.parametrize("rows_cap,max_ticks", [(3, 5), (7, 5)], ids=["rows3-events5", "rows7-events5"])
def test_policy_fuzz_resumed_windows(fuzz_cases, engine, rows_cap, max_ticks):
    """every fourth random case, resumed launch after launch: a launch ends when its row window is full (3 rows, 5
    events allowed) or when its event budget is spent (5 events, 7 rows allowed); every launch before the last one
    of a replica stops exactly there"""
    cases, refs = fuzz_cases
    sub = list(range(0, len(cases), 4))
    wins = []
    got = _run([(cases[i].cluster, cases[i].policy, cases[i].table) for i in sub], engine=engine, rows_cap=rows_cap,
               max_ticks=max_ticks, windows=wins)
    for i, g, w in zip(sub, got, wins):
        _assert_same(refs[i], g, f"seed {cases[i].seed} {cases[i].name} (resumed)")
        assert all(k == min(rows_cap, max_ticks) for k in w), (cases[i].seed, w)
    assert sum(len(w) for w in wins) > 100                    # most replicas took several launches


def _policy(name, table, **kw):
    from gpuschedule_b200 import capi, policies
    if name == "gittins":
        kw.setdefault("gittins_delta", 200)
        return capi.make_policy("gittins", gittins_table=policies.build_gittins_table(policies.gittins_samples(table), kw["gittins_delta"]), **kw)
    if name in ("dlas", "dlas-gpu"):
        kw.setdefault("num_queue", 3)
        kw.setdefault("queue_limit", [4, 30])
    return capi.make_policy(name, **kw)


def _table(arrive, minutes, gpus, seed=1, gpc=1):
    from gpuschedule_b200 import ingest, tracegen
    n = len(arrive)
    cols = tracegen.synth_columns(n, seed=seed, gpu_per_container=gpc)
    cols.pop("model")
    cols["normalized_time"] = np.asarray(arrive, dtype=np.int64) * 10000
    cols["minutes"] = np.asarray(minutes, dtype=np.float64)
    cols["used_gpus"] = np.asarray(gpus, dtype=np.int64)
    return ingest.table_from_columns(cols)


def _arrivals(rows):
    live = rows["running"].astype(np.int64) + rows["queued"] + rows["finished"]
    return np.diff(np.concatenate([[0], live]))


def _check_all(cases, tags):
    import oracle
    refs = [oracle.run_policy(*c) for c in cases]
    for engine in (0, 2):
        for ref, g, tag in zip(refs, _run(cases, engine=engine), tags):
            _assert_same(ref, g, f"{tag} engine {engine}")
    return refs


def test_arrival_bursts_around_chunk_sizes():
    """k jobs arrive at one tick for k = 31, 32, 33, 64, 65, 200 (the ballot loop that counts a run of arrivals 32 at a
    time), twice, on a cluster they overfill, under every policy"""
    from gpuschedule_b200 import capi
    rng = np.random.default_rng(11)
    cluster = capi.make_cluster(num_switch=1, num_node_p_switch=5, num_gpu_p_node=8, gpu_memory_capacity=16)
    cases, tags, sizes = [], [], []
    for k in (31, 32, 33, 64, 65, 200):
        arrive = np.concatenate([np.zeros(k, dtype=np.int64), np.full(k, 6), 20 + np.arange(10)])
        n = len(arrive)
        table = _table(arrive, np.round(rng.uniform(1.0, 40.0, size=n), 3), rng.choice([1, 2, 4, 8], size=n), seed=k)
        for name in POLICIES:
            cases.append((cluster, _policy(name, table), table))
            tags.append(f"burst {k} {name}")
            sizes.append(k)
    refs = _check_all(cases, tags)
    for ref, k, tag in zip(refs, sizes, tags):
        a = _arrivals(ref.rows)
        assert a[0] == k and (a == k).sum() >= 2, tag
        assert int(ref.rows["queued"].max()) > 0, tag


def test_long_end_lists_and_ties_with_bursts():
    """40 / 70 / 100 one-GPU jobs that start together and end together (more than 32, two and three chunks of the end
    list), each end tied with the next burst's arrival (quirk Q25: the start event inherits the end list), with
    dlas queue jumps and gittins service quanta between the tie and the start event"""
    from gpuschedule_b200 import capi
    cluster = capi.make_cluster(num_switch=1, num_node_p_switch=8, num_gpu_p_node=16)      # 128 GPUs
    cases, tags = [], []
    for k in (40, 70, 100):
        arrive = np.concatenate([np.full(k, 10 * b) for b in range(4)])
        table = _table(arrive, np.full(len(arrive), 20.0), np.ones(len(arrive), dtype=np.int64), seed=k)
        for name in POLICIES:
            jumps = {"sjf": [], "dlas": [{"queue_limit": [4, 7]}], "dlas-gpu": [{"queue_limit": [4, 7]}], "gittins": [{"gittins_delta": 5}]}
            for extra in [{}] + jumps[name]:
                cases.append((cluster, _policy(name, table, **extra), table))
                tags.append(f"ends {k} {name} {extra}")
    refs = _check_all(cases, tags)
    for ref, tag in zip(refs, tags):
        a = _arrivals(ref.rows)
        d = np.diff(np.concatenate([[0], ref.rows["finished"].astype(np.int64)]))
        assert ((d > 32) & (a > 0)).any(), tag            # a long end list completed on the tick of a burst
        assert ((d > 32) & (a == 0)).any(), tag           # and the last one on its own


def _overflow_run(engine):
    """(oracle results, per replica (rows, recs, order, stats), device summaries) of the overflow case under sjf,
    dlas-gpu and gittins in one handle"""
    import oracle
    from gpuschedule_b200 import capi
    cluster, table = overflow_case()
    pols = overflow_policies(table)
    refs = {name: oracle.run_policy(cluster, pol, table) for name, pol in pols.items()}
    for name, ref in refs.items():
        assert (ref.rows["pend_sum"] > INT32_MAX).any(), name
    with capi.Engine(device=0, nsims=len(pols)) as eng:
        eng.set_engine(engine)
        for i, pol in enumerate(pols.values()):
            eng.config(i, cluster, pol)
            eng.load_trace(i, table)
        rows = eng.run_all()
        summ = eng.summarize()
        got = [(rows[i], *eng.fetch_jobs(i), eng.stats(i)) for i in range(len(pols))]
    return table, refs, got, summ


@pytest.mark.parametrize("engine", [0, 2], ids=["warp", "thread"])
def test_pending_time_sum_past_int32(engine):
    """32 jobs of 10^7 ticks on one GPU: a row's pend_sum passes 2^31 - 1 inside one chunk; rows and records against
    the oracle"""
    _, refs, got, _ = _overflow_run(engine)
    for (name, ref), g in zip(refs.items(), got):
        _assert_same(ref, g, name)


@pytest.mark.parametrize("engine", [0, 2], ids=["warp", "thread"])
def test_pending_time_summary_past_int32(engine):
    """the device summary of the same runs (pend_sum_sum, avg_pending_sum, ...) against a summary of the ORACLE's rows
    and records: a summary compared with the engine's own rows could not see a wrapped chunk sum"""
    from test_summary_cpu import assert_summary, job_columns, reference_summary
    table, refs, _, summ = _overflow_run(engine)
    for i, (name, ref) in enumerate(refs.items()):
        assert_summary(summ[i], reference_summary(ref.rows, *job_columns(table, ref.recs, ref.finish_order)), name)


def test_sjf_on_8192_nodes_beside_small_replicas():
    """sjf on 64 x 128 x 1 (8192 nodes): the sjf kernel's node table takes 64 KB of dynamic shared memory, past the
    48 KB that needs the opt-in.  The handle also holds the first two policy_case replicas (at most 200 jobs) of each
    policy -- small sjf, dlas, dlas-gpu and gittins clusters, which run in the same launches with that larger
    allocation -- and a second handle puts a fifo replica beside the 8192-node one"""
    import oracle
    from gpuschedule_b200 import capi, ingest, tracegen
    big = capi.make_cluster(num_switch=64, num_node_p_switch=128, num_gpu_p_node=1)
    cols = tracegen.synth_columns(700, seed=81, rate=1.0, gpu_choices=[1, 3, 64, 512, 2048], gpu_probs=[.3, .2, .2, .2, .1])
    cols.pop("model")
    table = ingest.table_from_columns(cols)
    cases, tags = [(big, capi.make_policy("sjf"), table)], ["sjf 8192 nodes"]
    seed, small = 0, []
    while len(small) < 2 * len(POLICIES):
        c = policy_case(seed, max_jobs=200)
        seed += 1
        if sum(x.name == c.name for x in small) < 2:
            small.append(c)
    for c in small:
        cases.append((c.cluster, c.policy, c.table))
        tags.append(f"seed {c.seed} {c.name}")
    small = capi.make_cluster(num_switch=1, num_node_p_switch=4)
    ftab = ingest.table_from_columns({k: v for k, v in tracegen.synth_columns(150, seed=82, rate=1.0).items() if k != "model"})
    refs = _check_all(cases, tags)
    assert int(refs[0].rows["busy_nodes"].max()) > 6144                # nodes past the first 48 KB of the table are used
    assert int(refs[0].rows["queued"].max()) > 32
    # and a fifo replica in a handle whose largest cluster has 8192 nodes
    fref = oracle.run_fifo(small, ftab)
    with capi.Engine(device=0, nsims=2) as eng:
        eng.config(0, big, capi.make_policy("sjf"))
        eng.load_trace(0, table)
        eng.config(1, small)
        eng.load_trace(1, ftab)
        rows = eng.run_all()
        recs, order = eng.fetch_jobs(0)
        _assert_same(refs[0], (rows[0], recs, order, eng.stats(0)), "sjf 8192 nodes beside fifo")
        frecs, forder = eng.fetch_jobs(1)
        assert rows[1].tobytes() == fref.rows.tobytes() and frecs.tobytes() == fref.recs.tobytes()
        assert np.array_equal(forder, fref.finish_order)
