"""The self-checks of tests/test_gpu_config_numerics.py beyond check_inputs, at K11 L300 and over key segments (also run without
a GPU by tests/test_config_numerics_inputs_cpu.py)."""
import torch

from tests.support.fp64 import BAR, query_codes, restate, sample_sets
from tests.support.sparse_cases import check_inputs, pick

TPP = 253        # tables per tag pass of the fused kernel (one-byte tags)
REG_CHUNKS = 256   # 32-candidate chunks a CTA keeps in registers per pass (8 per warp x 32 warps, 16 x 16 at 512 threads)


def seg_bounds(nseg, M):
    """(number of key segments, keys per segment) of tables over max_length M cut into nseg segments (mpig_create's rule)."""
    return nseg, (((M + nseg - 1) // nseg) + 63) & ~63


def pass_sets(c, codes, tpp=TPP):
    """Index lists of the keys that collide in >= 2 tables of ONE pass of tpp tables (the counts of the passes never combined),
    and per head the number of keys that collide exactly once in every pass and twice or more overall (`cross` keys)."""
    B, T, Hq = codes.shape[:3]
    G, L = c["G"], c["L"]
    sets, cross = [], torch.zeros((B, T, Hq), dtype=torch.int64)
    for b in range(B):
        kc = c["slots"][c["slot_of"][b]]["kcodes"]
        rows = []
        for t in range(T):
            heads = []
            for g in range(c["Hkv"]):
                qc = codes[b, t, g * G:(g + 1) * G].to(kc.device, torch.int16)
                any_pass = torch.zeros((G, kc.shape[-1]), dtype=torch.bool, device=kc.device)
                total = torch.zeros((G, kc.shape[-1]), dtype=torch.int64, device=kc.device)
                for p0 in range(0, L, tpp):
                    cnt = torch.zeros((G, kc.shape[-1]), dtype=torch.int64, device=kc.device)
                    for l0 in range(p0, min(L, p0 + tpp), 25):
                        l1 = min(l0 + 25, p0 + tpp, L)
                        cnt += (kc[g, None, l0:l1] == qc[:, l0:l1, None]).sum(dim=1)
                    any_pass |= cnt > 1
                    total += cnt
                for j in range(G):
                    heads.append(torch.nonzero(any_pass[j]).flatten())
                    cross[b, t, g * G + j] = int(((total[j] > 1) & ~any_pass[j]).sum())
            rows.append(heads)
        sets.append(rows)
    return sets, cross


def chunk_streams(c, codes, segs, tpp=TPP):
    """The largest number of 32-candidate chunks one CTA streams in one tag pass: per head, key segment and pass, the sum over
    the pass's tables of ceil(keys of the segment in the query's bucket / 32)."""
    B, T, Hq = codes.shape[:3]
    G, L, NB = c["G"], c["L"], 1 << c["K"]
    nseg, seg_len = segs
    worst = 0
    for b in range(B):
        kc = c["slots"][c["slot_of"][b]]["kcodes"]
        n = kc.shape[-1]
        seg = torch.arange(n, device=kc.device) // seg_len
        for g in range(c["Hkv"]):
            idx = (torch.arange(L, device=kc.device)[:, None] * nseg + seg[None]) * NB + kc[g].long()
            cnt = torch.bincount(idx.flatten(), minlength=L * nseg * NB).reshape(L, nseg, NB)
            for t in range(T):
                qc = codes[b, t, g * G:(g + 1) * G].to(kc.device).long()                          # (G, L)
                per = cnt[torch.arange(L, device=kc.device)[None, :, None], torch.arange(nseg, device=kc.device)[None, None, :],
                          qc[:, :, None]]                                                             # (G, L, nseg)
                ch = (per + 31) // 32
                for p0 in range(0, L, tpp):
                    worst = max(worst, int(ch[:, p0:p0 + tpp].sum(dim=1).max()))
    return worst


def _moved(c, o, alt):
    """Per checked head, max|alt - o| / max|o|."""
    a, b = pick(alt, c, None), pick(o, c, None)
    return (a - b).abs().amax(-1) / b.abs().amax(-1).clamp_min(1e-30)


def check_config_inputs(c, segs, label):
    """check_inputs of test_gpu_batch_numerics (the regime's property, its own perturbation, window_of_request_0, wrong_document,
    drop_sampled), then this file's: cross_pass and wrong_weights (K11 L300), drop_segment_s, window_of_head_0 (one kv-head).
    Prints how far each moves the output; returns the fp64 query codes."""
    moved = check_inputs(c)
    codes = query_codes(c["q"], c["hf"], c["K"], c["L"])[0]
    sets = sample_sets(c, codes)
    o = restate(c, codes, sets=sets)[0]
    extra = {}
    if c["L"] > TPP:
        psets, cross = pass_sets(c, codes)
        assert int(cross.min()) > 0, f"{label}: some head has no key hit once in each tag pass ({int(cross.min())})"
        extra["cross_pass"] = float(_moved(c, o, restate(c, codes, sets=psets)[0]).max())
        extra["wrong_weights"] = float(_moved(c, o, restate(dict(c, K=10, L=150), codes, sets=sets)[0]).max())
    nseg, seg_len = segs
    need = {"window_of_head_0"}
    if c["regime"] == "R1":   # the sampled half carries the mass, spread over the whole store
        need |= {"cross_pass", "wrong_weights"} | {f"drop_segment_{s}" for s in range(nseg)}
    elif c.get("dominant") is not None:   # one stored key carries the mass (R2, R4 "win": the window does)
        need.add(f"drop_segment_{c['dominant'] // seg_len}")
    for s in range(nseg):
        cut = [[[x[(x < s * seg_len) | (x >= (s + 1) * seg_len)] for x in row] for row in rows] for rows in sets]
        extra[f"drop_segment_{s}"] = float(_moved(c, o, restate(c, codes, sets=cut)[0]).max())
    if c["G"] == c["Hq"]:
        extra["window_of_head_0"] = float(_moved(c, o, restate(c, codes, "window_of_head_0", sets=sets)[0]).max())
    moved.update(extra)
    print(f"{label}: perturbations move the output by " + ", ".join(f"{k} {v:.2e}" for k, v in moved.items()))
    for name, v in extra.items():
        if name in need:
            assert v >= 10 * BAR, f"{label}: inputs are insensitive: '{name}' moves the output by {v:.2e} only"
    return codes
