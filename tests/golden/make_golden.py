"""Generate the golden vectors under tests/golden/ by running the UNMODIFIED reference operators.

The reference ships no golden vectors or seeds for this path (SURVEY.md 8(c): its tests are
property-style on unseeded random data), so these fixtures are produced by executing the reference's
own compiled operators (`oracle/_ref`, built from a reference checkout by oracle/build_ref.py) on seeded
inputs, where such a checkout exists.  The tests need only the fixtures.

    python tests/golden/make_golden.py          # rewrites tests/golden/*.npz and reference_signatures.json

Files
  small_chain.npz  B=2 Hq=4 Hkv=2 d=128 K=6 L=24 n=128 M=160: all inputs stored + reference outputs
                   of LSH.fill/batch_retrieve/get_mask and SparseAttentionServer.attention_wrapper,
                   plus one all-miss query row set (nnz = 0 edge).
  c1_chain.npz     BASELINE config[0]: 1 head, seq 4096, d 128, K 10, L 150 (M = 4224); inputs are
                   regenerated from seeds by magicpig_b200.synth (checksums stored), outputs stored.
  live_reference.npz  outputs of LSH.fill/batch_retrieve/get_mask on library/lsh/test.py-shaped cases and of
                   SparseAttentionServer.attention_wrapper on one case; inputs regenerated from seeds by
                   live_probe_inputs / live_attention_inputs below (checksums stored).
  reference_signatures.json  the reference's Python API surface, read from its sources with `ast` / regexes:
                   LSHSparseAttnServer's methods (parameter names, literal defaults), the call sites in
                   models/llama.py and in LSHSparseAttnServer itself (positional count, keyword names), and the
                   pybind `.def` lists with the C++ member parameter names of lsh.LSH / SparseAttentionServer.
"""
from __future__ import annotations

import ast
import hashlib
import json
import os
import re
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from magicpig_b200 import synth  # noqa: E402
from oracle import ref_loader  # noqa: E402


def u16(t: torch.Tensor) -> np.ndarray:
    return t.contiguous().view(torch.int16).numpy().view(np.uint16)


def checksum(*tensors) -> str:
    h = hashlib.sha256()
    for t in tensors:
        t = t.contiguous()
        if t.dtype == torch.bfloat16:
            t = t.view(torch.int16)
        h.update(t.numpy().tobytes())
    return h.hexdigest()


def run_reference_chain(B, Hq, Hkv, d, K, L, n, M, key, value, key_norm, hash_func, query, qcodes=None):
    """key/value (B,Hkv,n,d) bf16, key_norm (B,Hkv,n), query (B,Hq,1,d) bf16 -> dict of reference outputs."""
    lsh_m, sa_m, flavour = ref_loader.load()
    kcodes = synth.hash_keys(key, hash_func, K, L)  # (B,Hkv,L,n) int16
    if qcodes is None:
        qcodes = synth.hash_queries_ref(query, hash_func, K, L)
    sc, si = kcodes.sort()
    R = lsh_m.LSH()
    R.alloc(K, L, 1, Hq, Hkv, B, M)
    for b in range(B):
        R.fill(0, b, sc[b].contiguous(), si[b].int().contiguous())
    results = torch.zeros((B * Hq, M), dtype=torch.int32)
    nnz = torch.zeros((B * Hq,), dtype=torch.int32)
    R.batch_retrieve(0, qcodes.contiguous(), results, nnz)
    mask = R.get_mask().clone().view(torch.uint8).reshape(B * Hq, M)
    S = sa_m.SparseAttentionServer()
    S.alloc(1, Hq, Hkv, d, B, M)
    for b in range(B):
        S.fill(0, b, key[b].contiguous(), value[b].contiguous(), key_norm[b].contiguous())
    out = torch.zeros((B * Hq, d), dtype=torch.bfloat16)
    mve = torch.zeros((2, B * Hq), dtype=torch.float32)
    q2 = query.reshape(B * Hq, d).contiguous()
    qn = q2.float().norm(p=2, dim=-1)
    S.attention_wrapper(0, K, L, out, mve, q2, qn, results, nnz)
    # results as sorted sets, flattened with offsets (order is unspecified by the reference)
    flat, offs = [], [0]
    for h in range(B * Hq):
        s = results[h, : nnz[h]].sort().values
        flat.append(s)
        offs.append(offs[-1] + int(nnz[h]))
    return dict(kcodes=kcodes.numpy(), qcodes=qcodes.numpy(), nnz=nnz.numpy(),
                results_sorted=torch.cat(flat).numpy() if flat else np.zeros(0, np.int32),
                results_offsets=np.array(offs, np.int64), mask=mask.numpy(), out_bf16=u16(out), mve=mve.numpy(),
                flavour=np.array(flavour))


def make_small():
    B, Hq, Hkv, d, K, L, n, M = 2, 4, 2, 128, 6, 24, 128, 160
    hf = synth.make_hash_func(d, K, L, seed=10)
    q = synth.make_query(B, Hq, d, seed=11)
    key, value, kn, avg = synth.make_kv(B, Hkv, n, d, seed=12, dist="gauss")
    ref = run_reference_chain(B, Hq, Hkv, d, K, L, n, M, key, value, kn, hf, q)
    # nnz = 0 edge: a query whose codes are all NB-1 XOR the majority never collides twice
    # (constructed: use codes no key carries in that table)
    kc = torch.from_numpy(ref["kcodes"])  # (B,Hkv,L,n)
    miss = torch.zeros((B * Hq, L), dtype=torch.int32)
    for h in range(B * Hq):
        b, g = h // Hq, (h % Hq) // (Hq // Hkv)
        for l in range(L):
            present = set(kc[b, g, l].tolist())
            miss[h, l] = next(c for c in range(1 << K) if c not in present)
    ref0 = run_reference_chain(B, Hq, Hkv, d, K, L, n, M, key, value, kn, hf, q, qcodes=miss)
    assert int(ref0["nnz"].sum()) == 0
    np.savez_compressed(
        os.path.join(HERE, "small_chain.npz"),
        dims=np.array([B, Hq, Hkv, d, K, L, n, M]), hash_func=u16(hf), query=u16(q), key=u16(key), value=u16(value),
        key_norm=kn.numpy(), avg_k=u16(avg), miss_qcodes=miss.numpy(), miss_nnz=ref0["nnz"], miss_out_bf16=ref0["out_bf16"],
        miss_lse2=ref0["mve"][1], **ref)
    print("small_chain: nnz", ref["nnz"].tolist())


def make_c1():
    B, Hq, Hkv, d, K, L, n = 1, 1, 1, 128, 10, 150, 4096
    M = n + 128
    hf = synth.make_hash_func(d, K, L, seed=0)
    q = synth.make_query(B, Hq, d, seed=1)
    key, value, kn, avg = synth.make_kv(B, Hkv, n, d, seed=2, dist="clustered", q_dirs=q.reshape(B, Hq, d)[:, :1].float())
    ref = run_reference_chain(B, Hq, Hkv, d, K, L, n, M, key, value, kn, hf, q)
    ref.pop("kcodes")
    ref.pop("mask")
    np.savez_compressed(os.path.join(HERE, "c1_chain.npz"), dims=np.array([B, Hq, Hkv, d, K, L, n, M]),
                        input_sha256=np.array(checksum(hf, q, key, value, kn)), **ref)
    print("c1_chain: nnz", ref["nnz"].tolist(), "sha", checksum(hf, q, key, value, kn)[:16])


# library/lsh/test.py's own case shapes: (K, L, seq, delta, group, bsz)
LIVE_PROBE_CASES = [(4, 50, 1024, 128, 4, 1), (8, 100, 1024, 128, 8, 2), (8, 50, 4096, 1024, 4, 1)]


def live_probe_inputs(K, L, seq, delta, group, bsz):
    """-> codes int16 (bsz, Hkv, L, seq), query int32 (bsz*Hq, L), Hq, Hkv, M"""
    g = torch.Generator().manual_seed(K * 1000 + L)
    Hq = 32
    Hkv = Hq // group
    NB, M = 1 << K, seq + delta
    codes = torch.randint(0, NB, (bsz, Hkv, L, seq), generator=g, dtype=torch.int16)
    query = torch.randint(0, NB, (bsz * Hq, L), generator=g, dtype=torch.int32)
    return codes, query, Hq, Hkv, M


def live_attention_inputs():
    """-> dims (B, Hq, Hkv, d, K, L, n, M), key, value (B, Hkv, n, d) bf16, key_norm, q (B*Hq, d) bf16, ind, nnz"""
    g = torch.Generator().manual_seed(77)
    B, Hq, Hkv, d, K, L, n, M = 1, 8, 2, 128, 10, 150, 2048, 2048 + 128
    key = torch.randn((B, Hkv, n, d), generator=g).bfloat16()
    value = torch.randn((B, Hkv, n, d), generator=g).bfloat16()
    kn = key.norm(p=2, dim=-1).float()
    q = torch.randn((B * Hq, d), generator=g).bfloat16()
    nnz = torch.randint(1, n, (B * Hq,), generator=g).int()
    ind = torch.zeros((B * Hq, M), dtype=torch.int32)
    for h in range(B * Hq):
        ind[h, : nnz[h]] = torch.randperm(n, generator=g)[: nnz[h]].int()
    return (B, Hq, Hkv, d, K, L, n, M), key, value, kn, q, ind, nnz


def reference_probe(lsh_m, K, codes, query, Hq, Hkv, M):
    """LSH.fill (sorted codes) + batch_retrieve + get_mask of the reference -> results (H, M), nnz (H,), mask uint8 (H, M)"""
    bsz, _, L, _ = codes.shape
    sc, si = codes.sort()
    R = lsh_m.LSH()
    R.alloc(K, L, 1, Hq, Hkv, bsz, M)
    for b in range(bsz):
        R.fill(0, b, sc[b].contiguous(), si[b].int().contiguous())
    results = torch.zeros((bsz * Hq, M), dtype=torch.int32)
    nnz = torch.zeros((bsz * Hq,), dtype=torch.int32)
    R.batch_retrieve(0, query, results, nnz)
    return results, nnz, R.get_mask().clone().view(torch.uint8).reshape(bsz * Hq, M)


def reference_attention(sa_m, dims, key, value, kn, q, ind, nnz):
    """SparseAttentionServer.fill + attention_wrapper of the reference -> out bf16 (H, d), mve (2, H)"""
    B, Hq, Hkv, d, K, L, n, M = dims
    S = sa_m.SparseAttentionServer()
    S.alloc(1, Hq, Hkv, d, B, M)
    S.fill(0, 0, key[0].contiguous(), value[0].contiguous(), kn[0].contiguous())
    out = torch.zeros((B * Hq, d), dtype=torch.bfloat16)
    mve = torch.zeros((2, B * Hq))
    S.attention_wrapper(0, K, L, out, mve, q, q.float().norm(p=2, dim=-1), ind, nnz)
    return out, mve


def make_live():
    lsh_m, sa_m, flavour = ref_loader.load()
    arrays = {"flavour": np.array(flavour)}
    for i, case in enumerate(LIVE_PROBE_CASES):
        codes, query, Hq, Hkv, M = live_probe_inputs(*case)
        results, nnz, mask = reference_probe(lsh_m, case[0], codes, query, Hq, Hkv, M)
        arrays.update({f"probe{i}_sha256": np.array(checksum(codes, query)), f"probe{i}_results": results.numpy(),
                       f"probe{i}_nnz": nnz.numpy(), f"probe{i}_mask": mask.numpy()})
    dims, key, value, kn, q, ind, nnz = live_attention_inputs()
    out, mve = reference_attention(sa_m, dims, key, value, kn, q, ind, nnz)
    arrays.update({"attn_sha256": np.array(checksum(key, value, kn, q, ind, nnz)), "attn_out_bf16": u16(out), "attn_mve": mve.numpy()})
    np.savez_compressed(os.path.join(HERE, "live_reference.npz"), **arrays)
    print("live_reference: probe nnz sums", [int(arrays[f"probe{i}_nnz"].sum()) for i in range(len(LIVE_PROBE_CASES))])


def _call_shape(node: ast.Call) -> dict:
    return {"nargs": len(node.args), "keywords": [k.arg for k in node.keywords]}


def reference_signatures(ref: str) -> dict:
    """The reference's API surface read from the sources of the checkout at `ref` (see reference_signatures.json)."""

    def read(path):
        with open(os.path.join(ref, path)) as f:
            return f.read()

    def find_class(tree, name):
        return next(n for n in ast.walk(tree) if isinstance(n, ast.ClassDef) and n.name == name)

    out = {}
    cls = find_class(ast.parse(read("models/attnserver.py")), "LSHSparseAttnServer")
    methods = {}
    for fn in (n for n in cls.body if isinstance(n, ast.FunctionDef)):
        args = [a.arg for a in fn.args.args]
        defaults = []
        for a, dflt in zip(args[len(args) - len(fn.args.defaults):], fn.args.defaults):
            try:
                defaults.append({"arg": a, "literal": True, "value": ast.literal_eval(dflt)})
            except ValueError:
                defaults.append({"arg": a, "literal": False, "value": None})   # e.g. torch.bfloat16
        methods[fn.name] = {"args": args, "defaults": defaults}
    out["attnserver_methods"] = methods
    owners = ("attn_server", "lsh_retriever")
    out["attnserver_operator_calls"] = [
        {"owner": n.func.value.attr, "method": n.func.attr, **_call_shape(n)} for n in ast.walk(cls)
        if isinstance(n, ast.Call) and isinstance(n.func, ast.Attribute) and isinstance(n.func.value, ast.Attribute)
        and n.func.value.attr in owners]
    calls = []
    for n in ast.walk(ast.parse(read("models/llama.py"))):
        if not isinstance(n, ast.Call):
            continue
        f = n.func
        if isinstance(f, ast.Name) and f.id == "LSHSparseAttnServer":
            calls.append({"method": "__init__", **_call_shape(n)})
        elif isinstance(f, ast.Attribute) and isinstance(f.value, ast.Attribute) and f.value.attr == "attention_server":
            calls.append({"method": f.attr, **_call_shape(n)})
    out["llama_calls"] = calls
    pybind = {}
    for cc, hdr, name in (("library/lsh/lsh.cc", "library/lsh/lsh.h", "LSH"),
                          ("library/sparse_attention/sparse_attention.cc", "library/sparse_attention/sparse_attention.h",
                           "SparseAttentionServer")):
        body = read(hdr)
        body = body[body.index(f"class {name}"):]
        body = body[: body.index("private:")]
        members = {}
        for m in re.finditer(r"(?:void|torch::Tensor|int)\s+([a-z_0-9]+)\(([^)]*)\);", body):
            params = [p.strip().split()[-1] for p in m.group(2).split(",") if p.strip()]
            members[m.group(1)] = [re.sub(r"_pt$", "", p) for p in params]   # without the `_pt` suffix of tensor arguments
        pybind[name] = {"defs": re.findall(r'\.def\("([a-z_0-9]+)"', read(cc)), "members": members}
    out["pybind"] = pybind
    return out


def make_signatures():
    from oracle.build_ref import REF
    out = reference_signatures(REF)
    with open(os.path.join(HERE, "reference_signatures.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print("reference_signatures: methods", sorted(out["attnserver_methods"]), "llama calls", len(out["llama_calls"]))


if __name__ == "__main__":
    torch.set_num_threads(4)
    make_small()
    make_c1()
    make_live()
    make_signatures()
