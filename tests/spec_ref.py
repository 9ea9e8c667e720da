"""Host twin of the speculative loop's acceptance rule (b200_generate_speculative, k_spec_accept).

target_next(ctx) and draft_next(ctx, i) give the next id after the id sequence ctx (prompt + ids so far + proposals);
draft_next also learns which proposal of the iteration it makes (1 .. n_draft), so a test can script a mismatch at a fixed
place.  Both must depend on their arguments only, as a model's choice depends only on the tokens before it (sampled: the
draw index is len(ctx) - len(prompt), the same for target and draft)."""


def plain(target_next, prompt, n_steps):
    """The plain generation loop: one target step per id."""
    ids = []
    for _ in range(n_steps):
        ids.append(target_next(list(prompt) + ids))
    return ids


def speculate(target_next, draft_next, prompt, n_steps, n_draft):
    """-> (ids, {"passes", "drafted", "accepted"}) of the speculative loop: step 0 is the prompt; each iteration the draft
    proposes d_1 .. d_k, the target chooses g_j after [t, d_1 .. d_j], and g_0 .. g_n are kept, n the largest j <= k with
    d_i == g_(i-1) for every i <= j, cut at the budget.  accepted counts every matching proposal, budget or not."""
    prompt = list(prompt)
    ids = [target_next(prompt)]
    stats = {"passes": 0, "drafted": 0, "accepted": 0}
    while len(ids) < n_steps:
        ctx = prompt + ids
        d = []
        for i in range(1, n_draft + 1):
            d.append(draft_next(ctx + d, i))
        g = [target_next(ctx + d[:j]) for j in range(n_draft + 1)]
        n = 0
        while n < n_draft and d[n] == g[n]:
            n += 1
        ids += g[:min(n + 1, n_steps - len(ids))]
        stats["passes"] += 1
        stats["drafted"] += n_draft
        stats["accepted"] += n
    return ids, stats
