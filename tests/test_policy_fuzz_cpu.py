"""Random cases for the event-driven policies (sjf / dlas / dlas-gpu / gittins) and CPU checks of the policy oracle
(oracle/policy_oracle.c) on them.

policy_case(seed) draws one cluster, one trace and one policy.  It aims at the places where the warp kernels of
gs_policy.cuh change path at a 32-entry chunk border: runs of more than 32 / 64 arrivals at one tick, more than 32
completions at one event (also on an end / start tie, quirk Q25), admission that runs out of GPUs inside a chunk,
gittins lists around multiples of 32 and 64, sjf node walks over node counts that are not multiples of 32, 64-GPU
nodes, slot-bound nodes (K = 0 included), jobs that leak (too big for a device) or are wider than the cluster, and
dlas queue limits of 2^31 and more.  tests/test_gpu_policy_fuzz.py runs the same cases on the GPU against the oracle;
tests/golden/fuzz_policy_reference.py pins the oracle to the reference's loop code on them.  Generator coverage below
counts, from the oracle's outputs, how often each of those edges occurs in the seed range the GPU test runs."""
import types

import numpy as np
import pytest

POLICIES = ("sjf", "dlas", "dlas-gpu", "gittins")
GPU_SEEDS = range(0, 240)                 # the seeds tests/test_gpu_policy_fuzz.py runs as one handle
OFTEN_M = (31, 32, 33, 63, 64, 65)        # node counts around a chunk of 32
GITTINS_DELTAS = (5, 20, 60, 200, 3250)
INT32_MAX = 2 ** 31 - 1


def _split_nodes(rng, m):
    """(num_switch, num_node_p_switch) with product m"""
    ds = [d for d in (1, 2, 3, 4) if m % d == 0]
    s = int(rng.choice(ds))
    return s, m // s


def policy_case(seed, max_jobs=600):
    """One random (cluster, trace, policy) as a namespace: seed, name, ckw (make_cluster keywords), pkw (make_policy
    keywords without the gittins table), gittins_form ('trace' / 'bisection' / 'one'), gittins_table ((data, index) or
    None), cluster, policy, table, step (the arrival flooring step, 1 = none)."""
    from gpuschedule_b200 import capi, ingest, policies, tracegen
    rng = np.random.default_rng(seed)
    name = POLICIES[int(rng.integers(0, 4))]
    sjf = name == "sjf"
    G = int(rng.choice([1, 2, 4, 8, 16, 64]))
    M = int(rng.choice(OFTEN_M)) if rng.random() < 0.45 else int(rng.integers(1, 141))
    ns, npp = _split_nodes(rng, M)
    ckw = dict(num_switch=ns, num_node_p_switch=npp, num_gpu_p_node=G, gpu_memory_capacity=int(rng.choice([16, 32])))
    if sjf and rng.random() < 0.5:        # cpu- or memory-bound nodes; 8 cpus or 50 GB give K = 0 (nothing can be placed)
        ckw.update(num_cpu_p_node=int(rng.choice([8, 24, 60, 128, 800], p=[.08, .3, .3, .22, .1])),
                   mem_p_node=int(rng.choice([50, 120, 300, 512, 4000], p=[.08, .3, .3, .22, .1])))
    gpc = int(rng.choice([1, 2, 4])) if sjf else 1
    total = M * G
    # job sizes scaled to the cluster so that large clusters are contended too
    top = max(1, total // int(rng.choice([1, 2, 4, 16])))
    base = sorted({1, 2, 4, 8} | {int(x) for x in (top, max(1, top // 2), G, 2 * G) if x >= 1})
    choices = sorted({int(x) * gpc for x in rng.choice(base, size=4)})
    if rng.random() < 0.25:               # wider than the cluster: never runs
        choices.append((total // gpc + 1 + int(rng.integers(0, 3))) * gpc)
    n = int(min(max_jobs, rng.integers(1, 601) if rng.random() < 0.8 else rng.integers(1, 40)))
    rate = float(rng.choice([0.2, 0.5, 1.0, 2.0, 4.0, 8.0]))
    cols = tracegen.synth_columns(n, seed=7000 + seed, rate=rate, gpu_per_container=gpc, gpu_choices=choices,
                                  gpu_probs=rng.dirichlet(np.ones(len(choices))),
                                  max_mem_mib=int(rng.choice([16384, 17000, 33500])))
    step = 1
    if rng.random() < 0.35:               # bursts: arrivals floored to a multiple of `step`, so that 33+ / 65+ share a tick
        step = int(rng.choice([5, 10, 20, 50, 100, 400]))
        arrive = cols["normalized_time"] // 10000
        cols["normalized_time"] = (arrive // step) * step * 10000
    minutes = cols["minutes"]
    if step > 1 and rng.random() < 0.5:   # lock step: a burst's jobs end together, on the tick of a later burst
        minutes = 2.0 * step * rng.choice([1, 1, 2, 3], size=n)
    elif rng.random() < 0.35:             # whole-tick durations: completions tie with arrivals
        minutes = np.round(minutes / 2.0) * 2.0
    if rng.random() < 0.3:                # durations below one tick (a job still runs for one)
        short = rng.random(n) < 0.3
        minutes = np.where(short, np.round(rng.uniform(0.05, 1.99, size=n), 3), minutes)
    cols["minutes"] = minutes
    cols.pop("model")
    table = ingest.table_from_columns(cols)
    pkw, form = {}, "trace"
    if name in ("dlas", "dlas-gpu"):
        nq = int(rng.integers(1, 9))
        inc = int(rng.choice([3, 20, 300, 3000]))          # increments of 1..2: one event demotes by several levels
        lim = np.cumsum(rng.integers(1, inc, size=nq - 1)).astype(np.float64)
        if nq > 1 and rng.random() < 0.25:                  # the top k limits 2^31, 2^31 + 10^9, ...
            k = int(rng.integers(1, nq))
            lim[nq - 1 - k:] = 2.0 ** 31 + 1e9 * np.arange(k)
        pkw = dict(num_queue=nq, queue_limit=[int(x) for x in lim])
    elif name == "gittins":
        pkw = dict(gittins_delta=int(rng.choice(GITTINS_DELTAS)))
        form = str(rng.choice(["trace", "trace", "bisection", "one"]))
    kw = dict(pkw)
    if name == "gittins":
        delta = float(pkw["gittins_delta"])
        samples = policies.gittins_samples(table)
        if form == "bisection":           # far-apart, partly non-integer sample positions: the kernel bisects
            data, index = policies.build_gittins_table(samples * 40000, delta * 40000)
            data = np.concatenate([np.sort(data[:-1] + 0.25 * (np.arange(len(data) - 1) % 2)), data[-1:]])
        elif form == "one":               # one sample: every attained service at or below it has the same index
            data, index = policies.build_gittins_table(samples[:1], delta)
        else:
            data, index = policies.build_gittins_table(samples, delta)
        kw["gittins_table"] = (data, index)
    return types.SimpleNamespace(seed=seed, name=name, ckw=ckw, pkw=pkw, gittins_form=form, step=step,
                                 gittins_table=kw.get("gittins_table"), cluster=capi.make_cluster(**ckw), policy=capi.make_policy(name, **kw), table=table)


def gittins_direct(case):
    """True when gs_config_sim tabulates this case's gittins table per whole unit (one load instead of a bisection)"""
    data = case.gittins_table[0]
    if len(data) < 2:
        return False
    last = float(data[-2])
    return 0.0 <= last < 8.0 * len(data) + 65536.0 and last < 67108864.0


def overflow_case():
    """32 one-GPU jobs of 10^7 ticks each on a 1 x 1 x 1 cluster: 31 of them wait while one runs, so a row's pend_sum
    passes 2^31 - 1 while the runnable list is still one chunk of 32"""
    from gpuschedule_b200 import capi, ingest, tracegen
    cols = tracegen.synth_columns(32, seed=5, gpu_choices=[1], gpu_probs=[1.0])
    cols["minutes"] = np.full(32, 2e7)
    table = ingest.table_from_columns(cols)
    return capi.make_cluster(num_switch=1, num_node_p_switch=1, num_gpu_p_node=1), table


def overflow_policies(table):
    from gpuschedule_b200 import capi, policies
    return {"sjf": capi.make_policy("sjf"),
            "dlas-gpu": capi.make_policy("dlas-gpu", num_queue=2, queue_limit=[1e9]),
            "gittins": capi.make_policy("gittins", gittins_table=policies.build_gittins_table(policies.gittins_samples(table)))}


def edges(case, ref):
    """the chunk-border edges one oracle run reaches: name -> bool"""
    t, rows = case.table, ref.rows
    M, G = case.cluster.n_nodes, case.cluster.num_gpu_p_node
    live = rows["running"].astype(np.int64) + rows["queued"] + rows["finished"]         # jobs arrived so far
    arrivals = np.diff(np.concatenate([[0], live]))
    done = np.diff(np.concatenate([[0], rows["finished"].astype(np.int64)]))
    listed = rows["running"].astype(np.int64) + rows["queued"]
    started = ref.recs["start"] >= 0
    e = {"burst33": bool((arrivals > 32).any()), "burst65": bool((arrivals > 64).any()),
         "end33": bool((done > 32).any()), "end33_tie": bool(((done > 32) & (arrivals > 0)).any()),
         "pend_wrap": bool((rows["pend_sum"] > INT32_MAX).any())}
    if case.name != "sjf":
        e["full_mid_list"] = bool(((rows["idle_gpus"] == 0) & (rows["queued"] > 0) & (listed > 32)).any())
    if case.name == "gittins":
        e["sort_len"] = {int(x) for x in np.unique(listed)} & {31, 32, 33, 63, 64, 65, 95, 96, 97, 127, 128, 129}
    if case.name == "sjf":
        K = min(case.ckw.get("num_cpu_p_node", 128) // 12, case.ckw.get("mem_p_node", 512) // 60)
        e["sjf_odd_m"] = M % 32 != 0 and bool(started.any())
        e["sjf_cross_node"] = bool((started & (t.gpus > G)).any())
        e["sjf_k0"] = K == 0
        e["sjf_gpc"] = int(t.gpu_per_task.max()) if t.n else 1
        fit = ((case.cluster.gpu_mem_cap_mib - 500) << 20)
        e["leak"] = bool((t.mem_bytes >= fit).any()) and not bool((started & (t.mem_bytes >= fit)).any())
    e["wider"] = bool((t.gpus > M * G).any()) and not bool((started & (t.gpus > M * G)).any())
    if case.name in ("dlas", "dlas-gpu"):
        lim = case.pkw["queue_limit"]
        e["big_limit"] = any(x >= 2 ** 31 for x in lim) and bool(started.any())
        e["tight_limits"] = len(lim) >= 2 and min(np.diff([0] + lim)) <= 2 and bool(started.any())
    return e


@pytest.fixture(scope="module")
def gpu_seed_runs():
    import oracle
    out = []
    for seed in GPU_SEEDS:
        case = policy_case(seed)
        out.append((case, oracle.run_policy(case.cluster, case.policy, case.table)))
    return out


def _event_identity(case, ref):
    """events = arrivals + completions + every start + every preemption; a job preempted after it joined an end list
    and then completed from it (quirk Q25) adds one preemption beyond resume - 1"""
    recs = ref.recs
    fin = np.zeros(case.table.n, dtype=bool)
    fin[ref.finish_order] = True
    resume = recs["preempt"].astype(np.int64)           # the record's `preempt` counts the job's (re)starts
    base = case.table.n + int(fin.sum()) + int(resume.sum()) + int((resume[fin] - 1).sum()) + int(resume[~fin].sum())
    return ref.events - base


@pytest.mark.parametrize("block", range(4))
def test_oracle_invariants_on_random_cases(block):
    """conservation, the event identity, start >= arrival, jct = ceil(duration) of finished jobs, on 400 seeds"""
    import oracle
    for seed in range(1000 + 100 * block, 1100 + 100 * block):
        case = policy_case(seed)
        t, ref = case.table, oracle.run_policy(case.cluster, case.policy, case.table)
        rows, recs = ref.rows, ref.recs
        total = case.cluster.n_nodes * case.cluster.num_gpu_p_node
        tag = (seed, case.name)
        order = ref.finish_order.tolist()
        assert len(set(order)) == len(order) and all(0 <= j < t.n for j in order), tag
        assert len(rows) == ref.ticks and ref.ticks >= 1, tag
        assert np.all(rows["busy_gpus"] + rows["idle_gpus"] == total) and np.all(rows["busy_gpus"] <= total), tag
        assert np.all(rows["busy_gpus"] >= 0) and np.all(rows["running"] >= 0) and np.all(rows["queued"] >= 0), tag
        live = rows["running"].astype(np.int64) + rows["queued"] + rows["finished"]
        assert np.all(np.diff(live) >= 0) and live[-1] == t.n, tag               # every job arrives, none is lost
        assert np.all(np.diff(rows["finished"]) >= 0) and rows["finished"][-1] == len(order), tag
        assert rows["running"][-1] == 0, tag
        if case.name == "sjf":
            assert np.all(rows["idle_nodes"] + rows["busy_nodes"] == case.cluster.n_nodes), tag
        else:
            assert np.all(rows["idle_nodes"] == case.cluster.n_nodes) and np.all(rows["busy_nodes"] == 0), tag
        need = np.maximum(1, np.ceil(t.duration)).astype(np.int32)
        fin = np.zeros(t.n, dtype=bool)
        fin[order] = True
        started = recs["start"] >= 0
        assert np.all(recs["start"][started] >= t.arrive_tick[started]), tag
        assert np.all(started[fin]) and np.all(recs["jct"][fin] == need[fin]), tag
        assert np.all(recs["end"][fin] >= recs["start"][fin]) and np.all(recs["end"][~fin] == -1), tag
        assert np.all(recs["preempt"][fin] >= 1) and np.all(recs["preempt"][~started] == 0), tag
        if case.name == "sjf":           # no jump events, so no end list outlives its event: every job runs its full length
            assert np.all(recs["end"][fin] - recs["start"][fin] >= need[fin]), tag
        extra = _event_identity(case, ref)
        assert extra == 0 if case.name == "sjf" else 0 <= extra <= len(order), (tag, extra)
        assert np.all(rows["pend_max"][rows["queued"] == 0] == 0) and np.all(rows["pend_sum"][rows["queued"] == 0] == 0), tag


def test_generator_covers_the_chunk_edges(gpu_seed_runs):
    """every edge the GPU fuzz is meant to reach occurs, measured on the oracle's outputs of the GPU seed range"""
    from collections import Counter
    cnt, sort_lens, gpcs, forms, deltas = Counter(), set(), set(), Counter(), set()
    ms, gs = set(), set()
    for case, ref in gpu_seed_runs:
        cnt[case.name] += 1
        ms.add(case.cluster.n_nodes)
        gs.add(case.cluster.num_gpu_p_node)
        for k, v in edges(case, ref).items():
            if k == "sort_len":
                sort_lens |= v
            elif k == "sjf_gpc":
                gpcs.add(v)
            elif v:
                cnt[k] += 1
        if case.name == "gittins":
            forms[case.gittins_form if case.gittins_form != "trace" else ("direct" if gittins_direct(case) else "bisection")] += 1
            deltas.add(case.pkw["gittins_delta"])
        cnt["n_max"] = max(cnt["n_max"], case.table.n)
        cnt["short"] += int((case.table.duration < 1).any())
        cnt["whole"] += int(case.table.n > 0 and (case.table.duration == np.floor(case.table.duration)).all())
        cnt["rate_sat"] += int(case.table.n > 32 and ref.rows["queued"].max() > 32)
    for p in POLICIES:
        assert cnt[p] >= 45, (p, cnt)
    need = {"burst33": 30, "burst65": 20, "end33": 5, "end33_tie": 3, "full_mid_list": 60, "sjf_odd_m": 20,
            "sjf_cross_node": 20, "sjf_k0": 3, "leak": 20, "wider": 40, "big_limit": 15, "tight_limits": 20,
            "short": 50, "whole": 50, "rate_sat": 100}
    for k, lo in need.items():
        assert cnt[k] >= lo, (k, cnt[k], lo, dict(cnt))
    assert cnt["n_max"] >= 500
    assert sort_lens >= {31, 32, 33, 63, 64, 65}, sorted(sort_lens)
    assert gpcs >= {1, 2, 4}, gpcs
    assert forms["direct"] >= 10 and forms["bisection"] >= 10 and forms["one"] >= 10, forms
    assert deltas == set(GITTINS_DELTAS), deltas
    assert gs == {1, 2, 4, 8, 16, 64} and len(ms & set(OFTEN_M)) == len(OFTEN_M) and max(ms) > 128, (gs, sorted(ms))


def test_overflow_case_sums_pending_time_past_int32():
    """the case the warp kernels' 32-bit chunk sum of pending times got wrong: a row's pend_sum > 2^31 - 1 while at
    most 32 jobs are runnable (one chunk), under sjf, dlas-gpu and gittins alike"""
    import oracle
    cluster, table = overflow_case()
    assert table.n == 32 and np.all(table.duration == 1e7)
    for name, pol in overflow_policies(table).items():
        ref = oracle.run_policy(cluster, pol, table)
        listed = ref.rows["running"].astype(np.int64) + ref.rows["queued"]
        assert listed.max() <= 32, name
        big = ref.rows["pend_sum"] > INT32_MAX
        assert big.sum() >= 5 and int(ref.rows["pend_sum"].max()) > 2 ** 31 + 2 ** 27, (name, int(ref.rows["pend_sum"].max()))
        # each waiting job's pending time is still an int
        assert int(ref.rows["pend_max"].max()) < INT32_MAX, name
        assert sorted(ref.finish_order.tolist()) == list(range(32)), name
