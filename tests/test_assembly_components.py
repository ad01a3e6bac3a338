"""Host-side model of the component-parallel get_humans that paf_limbs_kernel runs (hyperpose_b200/csrc/paf_parser.cu, phase d),
checked against the oracle's strictly sequential restatement of src/paf.cpp:146-232 on the oracle's own peaks / connections.

The claim the CUDA path rests on: a connection can only touch (paf.cpp:33-36) a partial human that holds one of its two peaks, so
the partial humans of different connected components of the (peaks, connections) graph never interact; replaying every component
on its own (global connection order inside it) and ordering the survivors by the index of the connection that CREATED them gives
the reference's vector -- except for frames in which a merge fabricates a peak id (`parts[i] += other.parts[i] + 1` with both set and
one id 0, paf.cpp:185-193), which are detected and left to the sequential path."""
import numpy as np
import pytest

import oracle
from oracle.binding import HUMAN_REC
from hyperpose_b200 import synthetic as syn

PAIRS = [(1, 2), (1, 5), (2, 3), (3, 4), (5, 6), (6, 7), (1, 8), (8, 9), (9, 10), (1, 11),
         (11, 12), (12, 13), (1, 0), (0, 14), (14, 16), (0, 15), (15, 17), (2, 16), (5, 17)]   # src/coco.hpp:32-52
f32 = np.float32


def _components(conns):
    """union-find over the end points of the connection list; returns the component id of every connection"""
    parent = {}

    def find(x):
        while parent.setdefault(x, x) != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x

    for _, c1, c2, _ in conns:
        a, b = find(c1), find(c2)
        if a != b:
            parent[max(a, b)] = min(a, b)
    return [find(c1) for _, c1, _, _ in conns]


def component_parallel_humans(orc, UW, UH):
    """-> HUMAN_REC array, or None when a merge would fabricate an id (the CUDA path then takes a sequential path)"""
    psc = orc["peaks"]["score"]
    conns = [(pair, int(c["cid1"]), int(c["cid2"]), f32(c["score"])) for pair in range(19) for c in orc["conns"][pair]]
    comp = _components(conns)
    survivors = []
    for root in sorted(set(comp)):
        humans = []   # dicts in creation order; dead ones stay in place
        for gi, (pair, c1, c2, sc) in enumerate(conns):
            if comp[gi] != root:
                continue
            p1, p2 = PAIRS[pair]
            touch = [h for h in humans if h["np"] >= 0 and (h["parts"][p1] == c1 or h["parts"][p2] == c2)][:2]
            if not touch:
                if pair <= 16:
                    parts = [-1] * 18
                    parts[p1], parts[p2] = c1, c2
                    humans.append({"parts": parts, "np": 2, "score": f32(f32(psc[c1] + psc[c2]) + sc), "made": gi})
            elif len(touch) == 1:
                h = touch[0]
                if h["parts"][p2] != c2:
                    h["parts"][p2] = c2
                    h["np"] += 1
                    h["score"] = f32(h["score"] + f32(psc[c2] + sc))
            else:
                h, o = touch
                if not any(a > 0 and b > 0 for a, b in zip(h["parts"], o["parts"])):
                    if any(a >= 0 and b >= 0 for a, b in zip(h["parts"], o["parts"])):
                        return None
                    h["parts"] = [a + b + 1 for a, b in zip(h["parts"], o["parts"])]
                    h["np"] += o["np"]
                    h["score"] = f32(f32(h["score"] + o["score"]) + sc)
                    o["np"] = -1
                else:
                    h["parts"][p2] = c2
                    h["np"] += 1
                    h["score"] = f32(h["score"] + f32(psc[c2] + sc))
        survivors += [h for h in humans if h["np"] >= 4 and not f32(h["score"] / f32(h["np"])) < f32(0.4)]
    survivors.sort(key=lambda h: h["made"])
    out = np.zeros(len(survivors), HUMAN_REC)
    pk = orc["peaks"]
    for i, h in enumerate(survivors):
        out[i]["score"] = h["score"]
        for q, pid in enumerate(h["parts"]):
            if 0 <= pid < len(pk):
                out[i]["parts"][q] = (1, f32(pk["x"][pid]) / f32(UW), f32(pk["y"][pid]) / f32(UH), pk["score"][pid])
    return out


def _noisy_case(seed):
    rng = np.random.default_rng(seed)
    hf, wf = 30, 40
    conf, paf = syn.make_frame_tensors(seed, int(rng.integers(3, 9)), hf, wf)
    amp = float(rng.uniform(0.05, 0.25))
    conf = (conf + rng.random(conf.shape, dtype=np.float32) * amp).astype(np.float32)
    paf = (paf + (rng.random(paf.shape, dtype=np.float32) - 0.5) * 2 * amp).astype(np.float32)
    return conf, paf


def test_component_replay_equals_the_sequential_reference_order():
    checked = fallbacks = 0
    cases = [syn.make_frame_tensors(s, P, 46, 54) for s, P in [(1, 1), (2, 3), (3, 12), (4, 20)]]
    cases += [(c[i], p[i]) for c, p in [syn.make_batch_tensors(1000, 4, (10, 20), 46, 82)] for i in range(4)]
    cases += [_noisy_case(s) for s in range(300, 324)]
    for conf, paf in cases:
        orc = oracle.oracle_process(conf, paf, peak_cap=1 << 18, conn_cap=1 << 14)
        got = component_parallel_humans(orc, 4 * conf.shape[1], 4 * conf.shape[2])
        if got is None:
            fallbacks += 1
            continue
        checked += 1
        assert got.tobytes() == orc["humans"].tobytes()
    assert checked >= 24 and fallbacks <= 8


def test_fabricated_id_is_detected():
    """pair 12 (neck 3 - nose 1) creates B = {neck 3, nose 1}; pair 13 (nose 0 - eye 4) creates A = {nose 0, eye 4}; a second pair-13
    connection (nose 1 - eye 4) touches both.  They share no part under the reference's `id > 0` test (A's nose is id 0), so the
    reference merges them and fabricates nose id 1 + 0 + 1 = 2; the model (like the CUDA path) reports the frame instead."""
    peaks = np.zeros(8, oracle.binding.PEAK_REC)
    peaks["score"] = 1.0
    mk = lambda rows: np.array(rows, oracle.binding.CONN_REC)
    conns = [mk([]) for _ in range(19)]
    conns[12] = mk([(3, 1, 1.0)])
    conns[13] = mk([(0, 4, 1.0), (1, 4, 1.0)])
    assert component_parallel_humans({"peaks": peaks, "conns": conns}, 100, 100) is None
    conns[13] = mk([(0, 4, 1.0)])      # without the linking connection nothing is fabricated
    assert component_parallel_humans({"peaks": peaks, "conns": conns}, 100, 100) is not None
