"""Sampling on the GPU: the sample_rows kernel (b200_op_sample) token for token against the oracle (oracle/sampling.py),
its distribution over many generation indices, and sampled requests through the engine and the serving shell."""
import json

import numpy as np
import pytest
import torch
from scipy import stats

from oracle.sampling import filter_mask, probs, sample_ref, scaled

pytestmark = pytest.mark.gpu
MARGIN, SLACK = 1e-4, 1e-6   # oracle coin flips: race top-2 margin, top-p boundary slack


def bf16_rows(S, V, seed, scale=3.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(S, V, generator=g) * scale).bfloat16()


def mixed_params(S, seed):
    rng = np.random.default_rng(seed)
    T = rng.choice([0.0, 0.0, 0.5, 0.8, 1.0, 1.5], S).astype(np.float32)
    k = rng.choice([0, -1, 1, 5, 50, 1000, 200000], S)
    p = rng.choice([1.0, 0.95, 0.9, 0.5, 0.1], S)
    seeds = [int(x) for x in rng.integers(0, 2 ** 63, S, dtype=np.int64)]
    n = rng.integers(0, 5000, S)
    return T, k, p, seeds, n


def check_against_oracle(lf, got, T, k, p, seeds, n):
    exempt = 0
    for i in range(len(got)):
        tok, margin, slack = sample_ref(lf[i], T[i], k[i], p[i], seeds[i], n[i])
        if got[i] != tok:
            assert margin < MARGIN or slack < SLACK, (i, got[i], tok, margin, slack, T[i], k[i], p[i])
            exempt += 1
    return exempt


@pytest.mark.parametrize("V", [512, 1000, 128256])
@pytest.mark.parametrize("S", [1, 7, 128, 300])
def test_sample_matches_oracle_token_for_token(V, S):
    from kubeai_b200 import ops
    logits = bf16_rows(S, V, seed=V + S)
    T, k, p, seeds, n = mixed_params(S, seed=S * 7 + V)
    d = logits.cuda()
    got = ops.sample(d, T, k, p, seeds, n).cpu().numpy()
    exempt = check_against_oracle(logits.float().numpy(), got, T, k, p, seeds, n)
    print(f"V={V} S={S}: {exempt} of {S} positions exempt as oracle coin flips")
    assert exempt <= max(1, S // 50)
    greedy = T < 1e-5
    assert np.array_equal(got[greedy], ops.argmax(d).cpu().numpy()[greedy])


def test_sample_is_a_function_of_the_row_and_its_parameters():
    from kubeai_b200 import ops
    S, V = 128, 128256
    logits = bf16_rows(S, V, seed=5).cuda()
    T, k, p, seeds, n = mixed_params(S, seed=6)
    a = ops.sample(logits, T, k, p, seeds, n)
    assert torch.equal(a, ops.sample(logits, T, k, p, seeds, n))
    perm = np.random.default_rng(7).permutation(S)
    b = ops.sample(logits[torch.from_numpy(perm).cuda()].contiguous(), T[perm], k[perm], p[perm],
                   [seeds[i] for i in perm], n[perm])
    assert torch.equal(b, a[torch.from_numpy(perm).cuda()])
    # all-greedy rows are the argmax bit for bit
    assert torch.equal(ops.sample(logits, 0.0), ops.argmax(logits))


@pytest.mark.parametrize("k,p", [(40, 1.0), (0, 0.9), (1, 1.0)])
def test_distribution_over_generation_indices(k, p):
    """One Llama-3-sized row drawn at 65536 values of n: never outside the oracle's kept set, chi-square against the
    oracle's probabilities (fixed seed: the outcome is deterministic), top_k 1 = the argmax."""
    from kubeai_b200 import ops
    V, N, chunk, T, seed = 128256, 65536, 4096, 0.7, 0x5EED_0F_5A3
    row = bf16_rows(1, V, seed=99, scale=2.0)[0]
    row[int(torch.argmax(row.float()))] = row.float().max() + 0.5      # a unique maximum
    lf = row.float().numpy()
    keep, _ = filter_mask(scaled(lf, T), k, p)
    want = probs(lf, T, k, p)
    block = row.cuda().expand(chunk, V).contiguous()
    draws = np.concatenate([ops.sample(block, T, k, p, seed, np.arange(c, c + chunk)).cpu().numpy()
                            for c in range(0, N, chunk)])
    assert keep[draws].all(), "a token outside the kept set"
    if k == 1:
        assert (lf == lf.max()).sum() == 1 and (draws == int(np.argmax(lf))).all()
        return
    idx = np.flatnonzero(keep)
    exp = want[idx] * N
    obs = np.bincount(draws, minlength=V)[idx].astype(np.float64)
    big = exp >= 5                                  # pool the bins too small for the chi-square approximation
    obs_b, exp_b = np.append(obs[big], obs[~big].sum()), np.append(exp[big], exp[~big].sum())
    if exp_b[-1] == 0:
        obs_b, exp_b = obs_b[:-1], exp_b[:-1]
    res = stats.chisquare(obs_b, exp_b * obs_b.sum() / exp_b.sum())
    print(f"k={k} p={p}: {keep.sum()} kept, {len(obs_b)} bins, chi2 p={res.pvalue:.3g}")
    assert res.pvalue > 1e-3


# ------------------------------------------------------------------ engine (mini model)
PROMPTS = [list(np.random.default_rng(40 + i).integers(0, 512, 9 + i)) for i in range(8)]
SPECS = [dict(temperature=0.0), dict(temperature=0.0, top_k=3, seed=9), dict(temperature=0.8, top_p=0.9, seed=1),
         dict(temperature=1.0, seed=2), dict(temperature=0.7, top_k=5, seed=3),
         dict(temperature=1.3, top_k=40, top_p=0.95, seed=4), dict(temperature=0.5, seed=2 ** 40 + 17),
         dict(temperature=1.0, top_p=0.5, seed=6)]
N_TOK = 10


def run_batch(specs, keep_logits, check=False):
    from kubeai_b200.engine import Engine, mini_config
    with Engine(mini_config()) as e:
        if keep_logits:
            e.set_keep_logits(True)
        rids = [e.submit(p, max_tokens=N_TOK, **sp) for p, sp in zip(PROMPTS, specs)]
        outs = [[] for _ in rids]
        exempt = 0
        for step in range(N_TOK):
            ran, info = e.step()
            assert ran and info.sampled == len(rids)      # every request samples in every step, in submission order
            rows = e.read_logits(len(rids)) if check else None
            for i, r in enumerate(rids):
                toks = e.poll(r).tokens
                assert len(toks) == 1
                outs[i] += toks
                if check:
                    sp = specs[i]
                    T = sp.get("temperature", 0.0)
                    if T < 1e-5:
                        assert toks[0] == int(np.argmax(rows[i])), (i, step)
                        continue
                    tok, margin, slack = sample_ref(rows[i], T, sp.get("top_k", 0), sp.get("top_p", 1.0), sp["seed"], step)
                    if toks[0] != tok:
                        assert margin < MARGIN or slack < SLACK, (i, step, toks[0], tok, margin, slack)
                        exempt += 1
        if check:
            print(f"engine: {exempt} of {N_TOK * len(rids)} positions exempt")
            assert exempt <= 1
        return outs


def test_engine_sampled_batch_matches_oracle_and_is_reproducible():
    a = run_batch(SPECS, keep_logits=True, check=True)
    assert a == run_batch(SPECS, keep_logits=True)            # a fresh engine, the same streams
    assert a == run_batch(SPECS, keep_logits=False)           # the serving path (no kept logits) samples the same
    specs = [dict(s) for s in SPECS]
    specs[5]["seed"] = 12345
    c = run_batch(specs, keep_logits=False)
    assert c[5] != a[5] and [x for i, x in enumerate(c) if i != 5] == [x for i, x in enumerate(a) if i != 5]


def test_engine_refuses_bad_sampling_parameters():
    from kubeai_b200 import B200Error
    from kubeai_b200.engine import Engine, mini_config
    with Engine(mini_config()) as e:
        for bad in (dict(temperature=-1.0), dict(temperature=float("inf")), dict(temperature=float("nan")),
                    dict(top_p=1.5), dict(top_p=-0.1), dict(top_k=-2)):
            with pytest.raises(B200Error):
                e.submit([1, 2, 3], **bad)
        e.submit([1, 2, 3], temperature=0.9, top_p=0.0, top_k=-1)   # 0 and -1 are "off"


# ------------------------------------------------------------------ serving shell
def _server():
    from kubeai_b200.engine import Engine, mini_config
    from kubeai_b200.server import Server
    eng = Engine(mini_config(manual_step=0, max_model_len=1024, max_batched_tokens=512, num_kv_blocks=512))
    return Server([eng], model="mini", vocab=512, max_model_len=1024, enable_sampling=True), eng


def test_server_seeded_stream_is_reproducible_and_refusals_stay():
    body = dict(model="mini", messages=[{"role": "user", "content": "Tell me something."}], max_tokens=12, stream=True,
                temperature=0.8, top_p=0.9, seed=42)
    texts = []
    for _ in range(2):     # a fresh engine each time
        srv, eng = _server()
        r = srv.handle("POST", "/openai/v1/chat/completions", json.dumps(body))
        assert r.status == 200
        chunks = [json.loads(e) for e in r.sse_events()[:-1]]
        texts.append("".join(c["choices"][0]["delta"].get("content", "") for c in chunks if c["choices"]))
        for extra in ({"n": 2}, {"min_p": 0.1}):
            assert srv.handle("POST", "/openai/v1/chat/completions", json.dumps({**body, **extra})).status == 400
        srv.close()
        eng.close()
    assert texts[0] == texts[1] and len(texts[0]) > 0


def test_harness_with_temperature_in_process():
    from kubeai_b200.server import harness_config, harness_run
    srv, eng = _server()
    cfg = harness_config(request_model="mini", max_concurrent_threads=4, max_completion_tokens=5, synth_threads=4,
                         synth_mean_words=6, vocab=512, seed=3, temperature=0.8)
    r = harness_run(cfg, server=srv)
    srv.close()
    eng.close()
    assert r["failed_threads"] == 0, r["first_error"]
    assert r["completion_tokens"] == 5 * r["request_count"] > 0
