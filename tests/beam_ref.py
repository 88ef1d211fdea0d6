"""calm_b200_decode_beam's rule (include/calm_b200.h), restated with numpy float32 from each step's per-row K-best lists:
candidates, walk, pool, done, the last step's live beams and the output order.  The CPU rule tests check it by hand and by
brute force; the GPU tests replay a call's own candidate lists through it."""
import numpy as np

f32 = np.float32


def norm_table(max_new, length_penalty):
    """norm[L] = (float)pow((double)L, (double)length_penalty), L = 1 .. max_new (entry 0 unused)."""
    return [f32(1.0)] + [f32(float(L) ** float(length_penalty)) for L in range(1, max_new + 1)]


def n_candidates(num_beams, n_stop):
    return max(2, 1 + n_stop) * num_beams


class Pool:
    """At most B finished hypotheses; the entry rule and the eviction rule of the header."""

    def __init__(self, B):
        self.B, self.items, self.added = B, [], 0  # items: (score, order, tokens, lps, raw sum)

    def worst(self):
        return min(range(len(self.items)), key=lambda i: (self.items[i][0], self.items[i][1]))

    def add(self, score, tokens, lps, raw):
        if len(self.items) == self.B and not score > self.items[self.worst()][0]:
            return
        self.items.append((f32(score), self.added, list(tokens), list(lps), f32(raw)))
        self.added += 1
        if len(self.items) > self.B:
            del self.items[self.worst()]

    def ordered(self):
        return sorted(self.items, key=lambda h: (-float(h[0]), h[1]))


def replay(step_lists, B, stop=(), length_penalty=1.0, early_stopping=0, max_new=None):
    """Run the rule over step_lists[j] = (ids int[rows][K], lps float32[rows][K]), rows = 1 at step 0 and B after, until
    done, max_new steps or the lists run out (max_new defaults to their number).  Returns a dict: hyps (tokens, lps,
    score) best first, steps, anc (the ancestry the last step read, [B][max_new], -1 where unset), back[j] = [(parent,
    token, lp)] for the beams step j made, beams[j] = the token histories of step j's rows, live = those of the beams
    after the last step, and raw = the hypotheses' raw sums."""
    max_new = len(step_lists) if max_new is None else max_new
    stop = set(int(s) for s in stop)
    K = n_candidates(B, len(stop))
    norm = norm_table(max_new, length_penalty)
    pool = Pool(B)
    S = [f32(0)]  # each live row's sum
    hist = [([], [])]  # each live row's tokens and lps
    anc = np.full((B, max_new), -1, np.int64)
    anc[0, 0] = 0
    anc_read, back, beams = None, [], []
    done, j = False, 0
    while j < min(max_new, len(step_lists)) and not done:
        ids, lps = (np.asarray(x) for x in step_lists[j])
        rows = 1 if j == 0 else B
        assert ids.shape[0] >= rows and ids.shape[1] == K, f"step {j}: lists of shape {ids.shape}, want ({rows}, {K})"
        anc_read = anc.copy()
        beams.append([h[0] for h in hist])
        cands = []
        for b in range(rows):
            for r in range(K):
                lp = f32(lps[b, r])
                cands.append((f32(S[b] + lp), b, r, int(ids[b, r]), lp))
        cands.sort(key=lambda x: (-float(x[0]), x[1], x[2]))
        nS, nhist, made, parents = [], [], [], []
        for q, (c, b, r, tok, lp) in enumerate(cands[:K]):
            if len(made) == B:
                break
            if tok in stop:
                if q < B:
                    pool.add(f32(c / norm[max(1, j)]), hist[b][0] + [tok], hist[b][1] + [lp], c)
                continue
            nS.append(c), nhist.append((hist[b][0] + [tok], hist[b][1] + [lp])), made.append((b, tok, lp)), parents.append(b)
        back.append(made)
        if len(pool.items) == B:
            worst = pool.items[pool.worst()][0]
            done = bool(early_stopping) or bool(worst >= f32(nS[0] / norm[j + 1]))
        if j + 1 < max_new:
            new = np.full((B, max_new), -1, np.int64)
            for b, p in enumerate(parents):
                new[b, :j + 1] = anc[p, :j + 1]
                new[b, j + 1] = b
            anc = new
        S, hist = nS, nhist
        j += 1
    live = [h[0] for h in hist]
    if not done:
        for b in range(B):
            pool.add(f32(S[b] / norm[max_new]), hist[b][0], hist[b][1], S[b])
    hyps = [(np.asarray(t, np.int32), np.asarray(lp, np.float32), f32(s)) for s, _, t, lp, _ in pool.ordered()]
    return {"hyps": hyps, "steps": j, "anc": anc_read, "back": back, "beams": beams, "live": live, "raw": [h[4] for h in pool.ordered()]}


def fsum(lps):
    """Left-to-right fp32 sum from 0."""
    s = f32(0)
    for x in lps:
        s = f32(s + f32(x))
    return s
