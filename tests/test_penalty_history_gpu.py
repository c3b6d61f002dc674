"""The logits-edit token history on the GPU (kubeai_b200/csrc/penalties.cu): update_kernel through b200_op_penalize_update,
and the edit / restore pair through b200_op_penalize_slots, on record lists built by b200_op_penalty_list in buffers the
test owns.  After every launch the whole record buffer and every length are compared with oracle.penalties.records: the
records below lens[slot] exactly, the poison at and past lens[slot] (but for the one appended record) and every list the
launch does not name bit for bit.  Lists span the 256-record chunks of the shift, full lists, the engine's capacity bound
and long streams at Llama-3's vocabulary; logits rows differ from list slots throughout.  The engine part checks that
sampled tokens follow the oracle while lists hold more than 256 records, through preemption and n = 4 groups."""
import numpy as np
import pytest
import torch

from oracle.penalties import PEN_BIAS, PEN_PROMPT, PEN_STOP, edit, records, sample_ref

pytestmark = pytest.mark.gpu
V = 128256
MAX_LOGIT_BIAS = 1024          # B200_MAX_LOGIT_BIAS: bias ids per request, and stop ids of a request with min_tokens
NEVER = 1 << 30                # a min_tokens no test reaches: stop records stay in force


def poisoned(n_slots, cap, seed):
    """Record lists (ops.penalty_lists) full of random words, lens poisoned too: a test names only lists it built."""
    from kubeai_b200 import ops
    recs, lens = ops.penalty_lists(n_slots, cap)
    g = torch.Generator().manual_seed(seed)
    recs.copy_(torch.randint(-2 ** 31, 2 ** 31 - 1, recs.shape, generator=g, dtype=torch.int32))
    lens.fill_(-7)
    return recs, lens


def build(recs, lens, slot, prompt=(), output=(), logit_bias=None, stop_ids=(), min_tokens=NEVER, history=True):
    """List `slot` as the engine builds it at admission; returns the kwargs that name it to oracle.penalties.records."""
    from kubeai_b200 import ops
    row = dict(prompt=list(prompt), output=list(output), logit_bias=logit_bias, stop_ids=list(stop_ids),
               min_tokens=min_tokens, repetition_penalty=1.25 if history else 1.0)
    ops.penalty_list(recs, lens, slot, V, row)
    return dict(prompt=list(prompt), output=list(output), history=history, logit_bias=logit_bias, stop_ids=list(stop_ids),
                min_tokens=min_tokens)


def snapshot(recs, lens):
    torch.cuda.synchronize()
    return recs.cpu().numpy().copy(), lens.cpu().numpy().copy()


def check(recs, lens, before, want):
    """The buffers are `before` with list s replaced by want[s] (records [0, len) and the length) for each s in want."""
    r, n = snapshot(recs, lens)
    er, en = before[0].copy(), before[1].copy()
    for s, w in want.items():
        er[s, :len(w)] = w
        en[s] = len(w)
    bad = np.flatnonzero(n != en)
    assert bad.size == 0, ("lens", bad[:8], n[bad[:8]], en[bad[:8]])
    bad = np.argwhere(r != er)
    assert bad.size == 0, ("records", bad[:8].tolist(), r[tuple(bad[0][:2])], er[tuple(bad[0][:2])])


def hrow(row, slot, history=1, n_generated=0, min_tokens=NEVER, presence=0.5, frequency=0.25, repetition=1.25):
    """A (row, slot, presence, frequency, repetition, n_generated, min_tokens, history) launch row."""
    return (row, slot, presence, frequency, repetition, n_generated, min_tokens, history)


# ------------------------------------------------------------------ lists
def test_penalty_list_equals_records_and_refusals():
    from kubeai_b200 import B200Error, ops
    rng = np.random.default_rng(1)
    recs, lens = poisoned(6, 3000, 1)
    before = snapshot(recs, lens)
    want = {}
    cases = [dict(prompt=rng.integers(0, V, 900), output=rng.integers(0, 500, 700),
                  logit_bias={int(t): float(rng.standard_normal() * 120) for t in rng.integers(0, V, 300)},
                  stop_ids=rng.integers(0, V, 40), min_tokens=701),
             dict(prompt=rng.integers(0, 300, 50), output=rng.integers(0, 300, 20), stop_ids=[7, 8], min_tokens=20),
             dict(prompt=rng.integers(0, V, 100), logit_bias={3: 1e9, 4: -1e9, 5: 0.0}, history=False),
             dict()]
    for slot, c in zip((4, 0, 2, 5), cases):
        kw = build(recs, lens, slot, **c)
        want[slot] = records(**kw)
    assert len(want[4]) > 1500 and want[0][:, 3].tolist().count(PEN_STOP) == 0
    assert (want[2][:, 3] == PEN_BIAS).all() and want[2][:, 2].view(np.float32).tolist() == [100.0, -100.0, 0.0]
    check(recs, lens, before, want)
    # refused: a slot outside the buffer, an id outside [0, V), a list longer than cap, no room at all
    for slot, row, r in ((6, {}, recs), (-1, {}, recs), (1, dict(prompt=[V]), recs),
                         (1, dict(stop_ids=[-1], min_tokens=1), recs),
                         (1, dict(prompt=range(3001), repetition_penalty=1.2), recs),
                         (0, {}, torch.zeros(6, 0, 4, dtype=torch.int32, device="cuda"))):
        with pytest.raises(B200Error) as ei:
            ops.penalty_list(r, lens, slot, V, row)
        assert ei.value.code == -1, (slot, row)
    check(recs, lens, before, want)


def test_refusals_leave_the_lists_alone():
    from kubeai_b200 import B200Error, ops
    recs, lens = poisoned(4, 64, 2)
    kw = build(recs, lens, 1, prompt=[5, 9, 11])
    build(recs, lens, 2, output=[6])
    before = snapshot(recs, lens)
    logits = torch.zeros(3, 1000, dtype=torch.bfloat16, device="cuda")
    bad_updates = [([hrow(0, 4)], [1, 1, 1]),                    # slot outside [0, n_slots)
                   ([hrow(0, -1)], [1, 1, 1]),
                   ([hrow(0, 1), hrow(1, 1)], [1, 2, 3]),        # one slot twice in a launch
                   ([hrow(3, 1)], [1, 1, 1]),                    # a row outside the logits
                   ([hrow(0, 1)], [V, 1, 1]),                    # a sampled id outside [0, V)
                   ([hrow(0, 1)], [1, -1, 1]),
                   ([hrow(0, 0)], [1, 1, 1])]                    # list 0 has a poisoned length
    for rows, sampled in bad_updates:
        with pytest.raises(B200Error) as ei:
            ops.penalize_update(recs, lens, rows, sampled, V)
        assert ei.value.code == -1, rows
    with pytest.raises(B200Error) as ei:
        ops.penalize_update(recs[:, :0].contiguous(), lens, [hrow(0, 1)], [1, 1, 1], V)   # cap < 1
    assert ei.value.code == -1
    for rows in ([hrow(0, 4)], [hrow(3, 1)], [hrow(0, 1), hrow(0, 2)], [hrow(0, 0)]):   # slot, row, a row twice, length
        with pytest.raises(B200Error) as ei:
            ops.penalize_slots(logits, rows, recs, lens)
        assert ei.value.code == -1, rows
    with pytest.raises(B200Error) as ei:      # list 1 holds id 11, outside a 10-token vocabulary
        ops.penalize_slots(logits[:, :10].contiguous(), [hrow(0, 1)], recs, lens)
    assert ei.value.code == -1
    torch.cuda.synchronize()
    assert (logits == 0).all()
    check(recs, lens, before, {1: records(**kw)})


# ------------------------------------------------------------------ update_kernel
CAP = 5000
N0 = [0, 1, 255, 256, 257, 511, 512, 513, 1000, 4097, CAP - 1]


def chunk_cases():
    """(n0, pos): a list of n0 records (ids 2k + 1) and a new id 2 pos that goes to record pos: the first and second
    record, the edges of the highest chunk the shift moves (n - 257 .. n - 255), the last record and the end."""
    return [(n0, p) for n0 in N0 for p in sorted({0, 1, n0 - 257, n0 - 256, n0 - 255, n0 - 1, n0}) if 0 <= p <= n0]


def mixed_list(n0):
    """Token lists whose records are ids 2k + 1, k < n0, with every kind of record: prompt, generated (1 to 3 times),
    bias and stop."""
    ids = 2 * np.arange(n0) + 1
    k = np.arange(n0)
    out = np.repeat(ids[k % 4 == 1], 1 + (k[k % 4 == 1] % 3))
    return dict(prompt=ids[k % 4 == 0].tolist(), output=out.tolist(),
                logit_bias={int(i): float((i % 200) - 100) * 0.37 for i in ids[k % 4 == 2]}, stop_ids=ids[k % 4 == 3].tolist())


def test_insert_at_every_chunk_edge():
    from kubeai_b200 import ops
    cases = chunk_cases()
    rng = np.random.default_rng(3)
    n_slots = len(cases) + 3
    recs, lens = poisoned(n_slots, CAP, 3)
    slots = rng.permutation(n_slots)[:len(cases)]
    rows = rng.permutation(len(cases))
    kws = [build(recs, lens, int(s), **mixed_list(n0)) for s, (n0, _) in zip(slots, cases)]
    before = snapshot(recs, lens)
    assert [int(before[1][s]) for s in slots] == [n0 for n0, _ in cases]
    sampled = np.zeros(len(cases), dtype=np.int32)
    sampled[rows] = [2 * p for _, p in cases]
    ops.penalize_update(recs, lens, [hrow(int(r), int(s)) for r, s in zip(rows, slots)], sampled, V)
    want = {}
    for s, kw, (n0, p) in zip(slots, kws, cases):
        w = records(**{**kw, "output": kw["output"] + [2 * p]})
        assert len(w) == n0 + 1 and w[p, 0] == 2 * p
        want[int(s)] = w
    check(recs, lens, before, want)


def test_hits_and_rows_without_history():
    """A prompt-only id counts 0 -> 1 and keeps its flag; a generated id counts + 1; a bias-only and a stop-only id keep
    their flags and bias; rows with history 0 change nothing, hit or miss."""
    from kubeai_b200 import ops
    base = dict(prompt=[10, 20, 30], output=[20, 40, 40], logit_bias={50: -3.5, 30: 7.0, 70: 1.5}, stop_ids=[60, 50])
    hits = [(10, PEN_PROMPT, 1), (20, PEN_PROMPT, 2), (40, 0, 3), (70, PEN_BIAS, 1), (60, PEN_STOP, 1),
            (50, PEN_BIAS | PEN_STOP, 1), (30, PEN_PROMPT | PEN_BIAS, 1)]
    S = len(hits) + 2
    recs, lens = poisoned(S, 600, 4)
    kws = [build(recs, lens, s, **base) for s in range(S)]
    before = snapshot(recs, lens)
    rows = [hrow(S - 1 - s, s) for s in range(len(hits))] + [hrow(1, S - 2, history=0), hrow(0, S - 1, history=0)]
    sampled = [0] * S
    for s, (t, _, _) in enumerate(hits):
        sampled[S - 1 - s] = t
    sampled[1], sampled[0] = 20, 99          # history 0: a hit and a miss
    ops.penalize_update(recs, lens, rows, sampled, V)
    want = {}
    for s, (t, flags, count) in enumerate(hits):
        w = records(**{**kws[s], "output": kws[s]["output"] + [t]})
        rec = w[np.searchsorted(w[:, 0], t)]
        assert rec[3] == flags and rec[1] == count, (t, rec)
        want[s] = w
    check(recs, lens, before, want)           # the lists of the history-0 rows keep their bits


def random_lists(rng, recs, lens, slots, max_prompt):
    kws = {}
    for s in slots:
        n_p = int(rng.integers(0, max_prompt))
        kws[int(s)] = build(recs, lens, int(s), prompt=rng.integers(0, V, n_p).tolist(),
                            output=rng.integers(0, 3000, int(rng.integers(0, 40))).tolist(),
                            logit_bias={int(t): float(rng.standard_normal()) for t in rng.integers(0, V, 4)},
                            stop_ids=rng.integers(0, V, 2).tolist())
    return kws


def test_a_thousand_rows_per_launch_in_any_order():
    """1024 rows a launch, logits rows a permutation unrelated to the slots: the lists do not depend on the order of the
    rows, and each is its oracle list."""
    from kubeai_b200 import ops
    rng = np.random.default_rng(5)
    n_rows, n_slots, cap = 1024, 1100, 700
    recs, lens = poisoned(n_slots, cap, 5)
    slots = rng.permutation(n_slots)[:n_rows]
    kws = random_lists(rng, recs, lens, slots, 600)
    before = snapshot(recs, lens)
    rows = rng.permutation(n_rows)
    sampled = np.empty(n_rows, dtype=np.int32)
    for r, s in zip(rows, slots):
        seen = kws[int(s)]["prompt"] + kws[int(s)]["output"]
        sampled[r] = seen[int(rng.integers(0, len(seen)))] if seen and rng.random() < 0.5 else int(rng.integers(0, V))
    launch = [hrow(int(r), int(s)) for r, s in zip(rows, slots)]
    recs2, lens2 = recs.clone(), lens.clone()
    ops.penalize_update(recs, lens, launch, sampled, V)
    want = {int(s): records(**{**kws[int(s)], "output": kws[int(s)]["output"] + [int(sampled[r])]})
            for r, s in zip(rows, slots)}
    check(recs, lens, before, want)
    ops.penalize_update(recs2, lens2, [launch[i] for i in rng.permutation(n_rows)], sampled, V)
    torch.cuda.synchronize()
    assert torch.equal(recs2, recs) and torch.equal(lens2, lens)


def test_long_streams_at_llama3_vocab():
    """4096 consecutive launches over 64 lists (8 of them without history), a token per list each, half repeats of the
    list's own history and half fresh ids; checked against the oracle every 256 launches and at the end."""
    from kubeai_b200 import ops
    rng = np.random.default_rng(6)
    n_slots, steps, S = 64, 4096, 80
    recs, lens = poisoned(n_slots, 4700, 6)
    kws = random_lists(rng, recs, lens, range(n_slots), 512)
    before = snapshot(recs, lens)
    history = np.ones(n_slots, dtype=bool)
    history[rng.permutation(n_slots)[:8]] = False
    outs = {s: list(kws[s]["output"]) for s in range(n_slots)}
    pool = [np.array(kws[s]["prompt"] + kws[s]["output"] + [0], dtype=np.int64) for s in range(n_slots)]
    grown = [np.zeros(steps, dtype=np.int64) for _ in range(n_slots)]
    for step in range(steps):
        rows = rng.permutation(S)[:n_slots]
        sampled = rng.integers(0, V, S).astype(np.int32)
        repeat = rng.random(n_slots) < 0.5
        for s in range(n_slots):
            if repeat[s]:
                k = int(rng.integers(0, len(pool[s]) + step))
                sampled[rows[s]] = pool[s][k] if k < len(pool[s]) else grown[s][k - len(pool[s])]
            grown[s][step] = sampled[rows[s]]
            if history[s]:
                outs[s].append(int(sampled[rows[s]]))
        ops.penalize_update(recs, lens, [hrow(int(rows[s]), s, history=int(history[s]), n_generated=step)
                                         for s in range(n_slots)], sampled, V)
        if (step + 1) % 256 == 0:
            check(recs, lens, before, {s: records(**{**kws[s], "output": outs[s]}) for s in range(n_slots)})
    assert max(len(records(**{**kws[s], "output": outs[s]})) for s in range(n_slots)) > 2000


def test_full_list():
    """With n == cap a new id leaves the list and its length alone and an id already there is counted; n == cap - 1 takes
    one more."""
    from kubeai_b200 import ops
    cap = 300
    recs, lens = poisoned(4, cap, 7)
    ids = (3 * np.arange(cap) + 2).tolist()
    kws = [build(recs, lens, s, prompt=ids[:cap - (s == 2)], output=ids[:40]) for s in range(3)]
    before = snapshot(recs, lens)
    assert before[1][:3].tolist() == [cap, cap, cap - 1]
    ops.penalize_update(recs, lens, [hrow(2, 0), hrow(0, 1), hrow(1, 2)], [ids[17], 0, 1], V)   # row 2: a new id
    want = {0: records(**kws[0]), 1: records(**{**kws[1], "output": kws[1]["output"] + [ids[17]]}),
            2: records(**{**kws[2], "output": kws[2]["output"] + [0]})}
    assert len(want[2]) == cap and want[2][0, 0] == 0
    check(recs, lens, before, want)


@pytest.mark.parametrize("max_model_len", [256, 4096])
def test_engine_capacity_bound_holds_the_worst_request(max_model_len):
    """The engine sizes each list at pen_cap = max_model_len + 2 * B200_MAX_LOGIT_BIAS + 1 records (engine.cu).  The
    largest list a request can own: max_model_len distinct prompt and generated ids (the last sampled token makes the
    sequence max_model_len long), 1024 more bias ids, and 1024 more stop ids plus EOS under min_tokens.  That is exactly
    pen_cap records: every generated id, the last included, is recorded; one record less would drop the last."""
    from kubeai_b200 import ops
    pen_cap = max_model_len + 2 * MAX_LOGIT_BIAS + 1
    gen = 64
    rng = np.random.default_rng(max_model_len)
    ids = rng.permutation(V)[:pen_cap].tolist()
    prompt, outputs = ids[:max_model_len - gen], ids[max_model_len - gen:max_model_len]
    bias = {t: float(rng.standard_normal()) for t in ids[max_model_len:max_model_len + MAX_LOGIT_BIAS]}
    stops = ids[max_model_len + MAX_LOGIT_BIAS:]         # 1024 stop ids and EOS
    assert len(stops) == MAX_LOGIT_BIAS + 1
    for cap in (pen_cap, pen_cap - 1):
        recs, lens = poisoned(3, cap, cap)
        # slot 2 is admitted before its first token; slot 0 is readmitted (after a preemption) with half its output
        kw2 = build(recs, lens, 2, prompt=prompt, logit_bias=bias, stop_ids=stops, min_tokens=gen)
        kw0 = build(recs, lens, 0, prompt=prompt, output=outputs[:gen // 2], logit_bias=bias, stop_ids=stops,
                    min_tokens=gen)
        before = snapshot(recs, lens)
        for k in range(gen):
            rows = [hrow(1, 2, n_generated=k, min_tokens=gen)] + ([hrow(0, 0, n_generated=k, min_tokens=gen)]
                                                                 if k >= gen // 2 else [])
            ops.penalize_update(recs, lens, rows, [outputs[k], outputs[k]], V)
        def grown(kw, out):      # the stop records stay after min_tokens tokens exist: the list was built before
            return records(**{**kw, "output": out, "min_tokens": NEVER})
        full = grown(kw2, outputs)
        assert len(full) == pen_cap
        if cap == pen_cap:
            check(recs, lens, before, {2: full, 0: grown(kw0, outputs)})
        else:   # one short: the last generated id is lost, without an error
            check(recs, lens, before, {2: grown(kw2, outputs[:-1]), 0: grown(kw0, outputs[:-1])})


def test_edit_and_restore_follow_the_updates():
    """Each step edits logits rows (unrelated to the slots) from the lists the previous updates grew, bit for bit as
    oracle.penalties.edit, restores the raw bits, then adds each row's token.  Lists run up to cap records."""
    from kubeai_b200 import ops
    rng = np.random.default_rng(8)
    cap, S, steps = 9000, 9, 12
    recs, lens = poisoned(12, cap, 8)
    params = [dict(presence=0.5, frequency=0.25, repetition=1.3, min_tokens=NEVER),
              dict(presence=-1.0, frequency=-0.5, repetition=0.8, min_tokens=5),
              dict(presence=0.0, frequency=2.0, repetition=1.0, min_tokens=NEVER),
              dict(presence=2.0, frequency=0.0, repetition=2.0, min_tokens=0),         # no stop records
              dict(presence=0.0, frequency=0.0, repetition=1.0, min_tokens=7)]      # no history: bias and stops only
    slots = [11, 3, 7, 0, 5]
    rows = [4, 8, 0, 2, 6]
    specs = []
    perm = rng.permutation(V).tolist()
    n_full = cap - 2 * 40 - steps          # slot 11: distinct prompt, bias, stop and generated ids, exactly cap in all
    fresh = perm[n_full + 80:n_full + 80 + steps]
    for i, (s, p) in enumerate(zip(slots, params)):
        if i == 0:
            prompt = perm[:n_full]
            bias = {t: float(rng.standard_normal() * 30) for t in perm[n_full:n_full + 40]}
            stops = perm[n_full + 40:n_full + 80]
        else:
            prompt = rng.integers(0, V, int(rng.integers(100, 3000))).tolist()
            bias = {int(t): float(rng.standard_normal() * 30) for t in rng.integers(0, V, 40)}
            stops = rng.integers(0, V, 40).tolist()
        hist = p["presence"] != 0 or p["frequency"] != 0 or p["repetition"] != 1
        row = dict(prompt=prompt, logit_bias=bias, stop_ids=stops, min_tokens=p["min_tokens"],
                   presence_penalty=p["presence"], frequency_penalty=p["frequency"], repetition_penalty=p["repetition"])
        ops.penalty_list(recs, lens, s, V, row)
        specs.append(dict(prompt=prompt, output=[], bias=bias, stops=stops, hist=hist, **p))
    for step in range(steps):
        before = snapshot(recs, lens)
        raw = (torch.randn(S, V, generator=torch.Generator().manual_seed(step)) * 3).bfloat16().cuda()
        raw[:, 3] = float("-inf")
        raw_bits = raw.view(torch.int16).cpu().numpy()
        logits = raw.clone()
        launch = [hrow(r, s, history=int(sp["hist"]), n_generated=step, min_tokens=sp["min_tokens"], presence=sp["presence"],
                       frequency=sp["frequency"], repetition=sp["repetition"]) for r, s, sp in zip(rows, slots, specs)]
        edited = ops.penalize_slots(logits, launch, recs, lens)
        torch.cuda.synchronize()
        assert np.array_equal(logits.view(torch.int16).cpu().numpy(), raw_bits)     # the restore gives the raw bits back
        got = edited.view(torch.int16).cpu().numpy()
        untouched = np.setdiff1d(np.arange(S), rows)
        assert np.array_equal(got[untouched], raw_bits[untouched])
        for r, sp in zip(rows, specs):
            want = edit(raw[r].float().cpu().numpy(), prompt=sp["prompt"], output=sp["output"], presence=sp["presence"],
                        frequency=sp["frequency"], repetition=sp["repetition"], min_tokens=sp["min_tokens"],
                        stop_ids=sp["stops"], logit_bias=sp["bias"])
            bad = np.flatnonzero(got[r] != (want.view(np.uint32) >> 16).astype(np.uint16).view(np.int16))
            assert bad.size == 0, (step, r, bad[:5])
        # restore=False leaves the edits in place
        inplace = ops.penalize_slots(raw.clone(), launch, recs, lens, restore=False)
        assert torch.equal(inplace, edited)
        sampled = np.zeros(S, dtype=np.int32)
        for r, sp in zip(rows, specs):
            seen = sp["prompt"] + sp["output"]
            if r == rows[0]:
                sampled[r] = fresh[step]
            else:
                sampled[r] = int(rng.integers(0, V)) if rng.random() < 0.5 else seen[int(rng.integers(0, len(seen)))]
            sp["output"].append(int(sampled[r]))   # a list without history does not count it, but min_tokens does
        ops.penalize_update(recs, lens, launch, sampled, V)
        # stop records stay once built: the lists were built with min_tokens > 0 or without stops
        check(recs, lens, before, {s: records(prompt=sp["prompt"], output=sp["output"], history=sp["hist"],
                                              logit_bias=sp["bias"], stop_ids=sp["stops"] if sp["min_tokens"] else (),
                                              min_tokens=NEVER)
                                   for s, sp in zip(slots, specs)})
    assert int(lens[slots[0]]) == cap


# ------------------------------------------------------------------ the engine, lists past one chunk
def _edited_sample(row, prompt, out, sp, k):
    return sample_ref(edit(row, prompt=prompt, output=out, presence=sp.get("presence_penalty", 0.0),
                           frequency=sp.get("frequency_penalty", 0.0), repetition=sp.get("repetition_penalty", 1.0)),
                      sp.get("temperature", 0.0), 0, 1.0, sp.get("seed", 0), k)


ENGINE_SPECS = [dict(repetition_penalty=1.3, frequency_penalty=0.4, presence_penalty=0.3),
                dict(temperature=0.9, seed=3, repetition_penalty=1.2, frequency_penalty=0.2, presence_penalty=0.5),
                dict(repetition_penalty=0.9, frequency_penalty=-0.3, presence_penalty=0.8),
                dict(temperature=0.7, seed=8, repetition_penalty=1.5, frequency_penalty=1.0)]


def _check_tokens(toks, rows, prompts, specs):
    """Every token is the oracle's sample of edit(kept raw row, prompt, output so far); seeded rows whose race margin is
    a coin flip (< 1e-4) are exempt, at most 2 in all (test_penalties_gpu.py's rule)."""
    exempt = compared = 0
    for t, rs, p, sp in zip(toks, rows, prompts, specs):
        assert len(t) == len(rs)
        for k, tok in enumerate(t):
            want, margin, slack, mslack = _edited_sample(rs[k], p, t[:k], sp, k)
            if min(margin, slack, mslack) < 1e-4 and sp.get("temperature", 0.0) > 0:
                exempt += 1
                continue
            assert tok == want, (k, tok, want, sp)
            compared += 1
    assert exempt <= 2 and compared > 0
    return compared


def _long_prompts(n, seed):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 512, int(rng.integers(600, 900))).tolist() for _ in range(n)]


@pytest.mark.parametrize("pressed", [False, True])
def test_engine_lists_past_one_chunk(pressed):
    """Requests with 600-900-token prompts over the test model's 512 ids (lists of more than 300 records) and 64
    generated tokens; pressed: a KV pool too small for all four, so requests are preempted and their lists rebuilt from
    the host on readmission."""
    from kubeai_b200.engine import Engine, mini_config
    prompts = _long_prompts(4, 10)
    assert min(len(records(prompt=p)) for p in prompts) > 300
    N = 64
    blocks = 150 if pressed else 512
    with Engine(mini_config(max_model_len=1024, num_kv_blocks=blocks, max_batched_tokens=512)) as e:
        e.set_keep_logits(True)
        rids = [e.submit(p, max_tokens=N, **sp) for p, sp in zip(prompts, ENGINE_SPECS)]
        toks, rows = [[] for _ in rids], [[] for _ in rids]
        for _ in range(2000):
            ran, info = e.step()
            if not ran:
                break
            kept = e.read_logits(info.sampled) if info.sampled else None
            j = 0
            for i, r in enumerate(rids):      # sampled rows come in running order, which is submission order here
                t = e.poll(r).tokens
                assert len(t) <= 1
                if t:
                    rows[i].append(kept[j])
                    j += 1
                toks[i] += t
            assert j == info.sampled
        st = e.stats()
    assert all(len(t) == N for t in toks)
    assert (st.preemptions > 0) == pressed
    _check_tokens(toks, rows, prompts, ENGINE_SPECS)


def test_engine_group_members_keep_their_own_lists():
    """An n = 4 group over a long prompt: each member's list starts from the shared prompt and counts its own tokens."""
    from kubeai_b200.engine import Engine, mini_config
    prompt = _long_prompts(1, 11)[0]
    N, n = 64, 4
    sp = dict(temperature=0.9, repetition_penalty=1.3, frequency_penalty=0.5, presence_penalty=0.4)
    with Engine(mini_config(max_model_len=1024, num_kv_blocks=512, max_batched_tokens=512)) as e:
        e.set_keep_logits(True)
        rids = e.submit_n(prompt, n, max_tokens=N, seed=40, **sp)
        toks, rows = [[] for _ in rids], [[] for _ in rids]
        for _ in range(2000):
            ran, info = e.step()
            if not ran:
                break
            kept = e.read_logits(info.sampled) if info.sampled else None
            j = 0
            for i, r in enumerate(rids):     # the members in index order
                t = e.poll(r).tokens
                if t:
                    rows[i].append(kept[j])
                    j += 1
                toks[i] += t
            assert j == info.sampled
    assert all(len(t) == N for t in toks) and len({tuple(t) for t in toks}) == n
    _check_tokens(toks, rows, [prompt] * n, [dict(sp, seed=40 + i) for i in range(n)])
