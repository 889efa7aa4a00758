"""An exact restatement of falcon_perplexity (the reference's examples/falcon_perplexity/falcon_perplexity.cpp): the per-row score and
the chunk / batch / scored-range loop around it, with the float transcendentals passed in (sampler_twin.GLIBC or sampler_twin.CR).

Per row l[0..V) with target t (falcon_perplexity.cpp:12-26, 113-115):
    m = max l;  e[i] = expf(l[i] - m) (float);  S = (((0.0 + e[0]) + e[1]) + ...) + e[V-1] (double, sequential);
    p = (float) ((double) e[t] / S);  term = -logf(p)
np.add.accumulate is a sequential loop, so S rounds once per add in id order, as the reference's loop does.  twin(GLIBC) is held to the
reference's own softmax, twin(CR) to the device (b200_token_nll, b200_falcon_score, b200_falcon_perplexity), each bit for bit."""
import math
import numpy as np

f32 = np.float32


def prob(row, t, fn):
    """softmax(row)[t] as falcon_perplexity's softmax computes it"""
    l = np.asarray(row, f32)
    e = fn.exp(l - l.max())
    S = np.add.accumulate(np.concatenate(([0.0], e.astype(np.float64))))[-1]
    return f32(np.float64(e[t]) / S)


def term(p, fn):
    """-std::log(prob) on a float: +inf for p == 0"""
    return -fn.log(f32(p))[0]


def terms(logits, targets, fn):
    """the term of every row whose target is not -1; NaN elsewhere (float32 [rows])"""
    out = np.full(len(targets), np.nan, f32)
    for r, t in enumerate(targets):
        if t >= 0:
            out[r] = term(prob(logits[r], int(t), fn), fn)
    return out


def plan(n_tokens, n_ctx, n_batch):
    """falcon_perplexity.cpp:37-117: per chunk (start, [(n_past, n_tokens) of each batch], [(k, index into tokens of row k's target)]);
    the tail after the last whole chunk is dropped"""
    out = []
    for c in range(n_tokens // n_ctx):
        start = c * n_ctx
        batches = [(j * n_batch, min(n_ctx - j * n_batch, n_batch)) for j in range((n_ctx + n_batch - 1) // n_batch)]
        scored = [(k, start + k + 1) for k in range(min(512, n_ctx // 2), n_ctx - 1)]
        out.append((start, batches, scored))
    return out


def perplexity(tokens, n_ctx, n_batch, eval_all_logits, fn):
    """the whole loop: eval_all_logits(tokens of a batch, n_past) -> its logits [N][V] (every row, as falcon_eval with logits_all);
    -> (ppl after each chunk as float64, the terms in order as float32).  nll (double) += term in k order over all chunks so far."""
    tokens = np.asarray(tokens, np.int32)
    nll, count, ppl, out = 0.0, 0, [], []
    for start, batches, scored in plan(tokens.size, n_ctx, n_batch):
        logits = np.concatenate([eval_all_logits(tokens[start + p0:start + p0 + n], p0) for p0, n in batches])
        for k, ti in scored:
            x = term(prob(logits[k], int(tokens[ti]), fn), fn)
            nll += float(x)
            count += 1
            out.append(x)
        ppl.append(math.exp(nll / count))
    return np.array(ppl, np.float64), np.array(out, f32)


def accumulate(chunk_terms):
    """the loop's sums over given per-chunk terms -> ppl after each chunk (float64)"""
    nll, count, ppl = 0.0, 0, []
    for ts in chunk_terms:
        for x in ts:
            nll += float(f32(x))
            count += 1
        ppl.append(math.exp(nll / count))
    return np.array(ppl, np.float64)


def case_rows(V, seed=0):
    """named (row, target) cases: random rows, all-equal (p = 1/V), one dominant logit (its target and another), spreads that make most
    e[i] subnormal or 0, a target at the maximum, a target whose e is 0 (term +inf)"""
    rng = np.random.default_rng(seed + V)
    cases = []
    for i in range(3):
        r = (rng.standard_normal(V) * (1 + 3 * i)).astype(f32)
        cases.append(("random%d" % i, r, int(rng.integers(V))))
    cases.append(("equal", np.full(V, 1.5, f32), int(rng.integers(V))))
    r = (rng.standard_normal(V) * 0.5).astype(f32)
    d = int(rng.integers(V))
    r[d] = 40.0
    cases.append(("dominant", r, d))
    cases.append(("dominant_other", r, (d + 1) % V))
    for i, lo in enumerate((-200.0, -400.0)):
        r = rng.uniform(lo, 0.0, V).astype(f32)
        r[int(rng.integers(V))] = 0.0
        cases.append(("wide%d" % i, r, int(rng.integers(V))))
    r = (rng.standard_normal(V) * 2).astype(f32)
    cases.append(("target_max", r, int(np.argmax(r))))
    r = rng.uniform(-160.0, 0.0, V).astype(f32)
    r[0] = 0.0
    z = int(np.nonzero(r < -110.0)[0][0])
    cases.append(("target_e_zero", r, z))
    return cases
