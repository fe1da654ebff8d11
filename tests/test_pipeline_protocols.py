"""Random-interleaving exploration of the mbarrier protocols of the fused-attention kernel and the GEMM
(tests/pipeline_protocol_model.py).  CPU only.  The shipped protocols must run to completion with every data-hazard check
silent under thousands of schedules, and single-line mutations of them must be caught."""
import pytest

from pipeline_protocol_model import Hazard, variant1, variant2


@pytest.mark.parametrize("nb", [1, 2, 3, 4, 8])
def test_variant1_protocol_has_no_deadlock_or_hazard(nb):
    for seed in range(300):
        variant1(nb, seed).run()


@pytest.mark.parametrize("kst,vst", [(2, 1), (2, 2), (4, 3)])
def test_variant1_protocol_other_ring_depths(kst, vst):
    for seed in range(150):
        variant1(5, seed, kst=kst, vst=vst).run()


@pytest.mark.parametrize("nb,items", [(1, 1), (1, 3), (2, 2), (3, 3), (5, 2), (8, 2)])
def test_variant2_protocol_has_no_deadlock_or_hazard(nb, items):
    for seed in range(250):
        variant2(nb, items, seed).run()


@pytest.mark.parametrize("kst,vst", [(2, 1), (2, 2), (4, 3)])
def test_variant2_protocol_other_ring_depths(kst, vst):
    for seed in range(100):
        variant2(4, 3, seed, kst=kst, vst=vst).run()


def _mutant(old, new, which, args, seeds=120):
    """Runs the model with one line of its source replaced; returns how many schedules raised a Hazard."""
    import inspect

    import pipeline_protocol_model as m
    src = inspect.getsource(m)
    assert old in src
    ns = {}
    exec(compile(src.replace(old, new, 1), "attn_protocol_mutant", "exec"), ns)
    caught = 0
    for seed in range(seeds):
        try:
            ns[which](*args, seed).run()
        except ns["Hazard"]:
            caught += 1
    return caught


@pytest.mark.parametrize("label,old,new,which,args", [
    ("attention: K-empty barrier counting 7 of the 8 consumer warps", 'M.bar(f"KFULL{s}", 1); M.bar(f"KEMPTY{s}", 8)',
     'M.bar(f"KFULL{s}", 1); M.bar(f"KEMPTY{s}", 7)', "variant2", (3, 3)),
    ("attention: V-empty barrier counting 7 of the 8 consumer warps", 'M.bar(f"VFULL{s}", 1); M.bar(f"VEMPTY{s}", 8)',
     'M.bar(f"VFULL{s}", 1); M.bar(f"VEMPTY{s}", 7)', "variant1", (4,)),
    ("attention: Q-empty arrival before the item's last score product",
     '                        yield from score(ks, kc, wi, last)\n                        if last:\n'
     '                            M.bars["QEMPTY"].arrive()\n',
     '                        if last:\n                            M.bars["QEMPTY"].arrive()\n'
     '                        yield from score(ks, kc, wi, last)\n', "variant2", (3, 3)),
    ("attention: next Q loaded without waiting for Q-empty", '            yield M.wait("QEMPTY", (wi & 1) ^ 1)\n',
     '            pass\n', "variant2", (2, 3)),
    ("attention: pass 2 not waiting for the V block", '                    yield M.wait(f"VFULL{vs}", (vc // vst) & 1)\n',
     '', "variant2", (3, 3)),
    ("gemm: ring slot kb released instead of kb-1",
     'M.bars[f"empty{c}.{(kb - 1) % stages}"].arrive()', 'M.bars[f"empty{c}.{kb % stages}"].arrive()', "gemm", (2, 12)),
    ("gemm: slot released with two k-blocks of wgmma in flight", 'yield M.inflight_at_most(me, 1)',
     'yield M.inflight_at_most(me, 2)', "gemm", (2, 12)),
    ("gemm: empty barrier counting 7 of the 8 consumer warps", 'M.bar(f"full{c}.{s}", 1); M.bar(f"empty{c}.{s}", 8)',
     'M.bar(f"full{c}.{s}", 1); M.bar(f"empty{c}.{s}", 7)', "gemm", (2, 12)),
])
def test_model_is_sensitive_to_protocol_mutations(label, old, new, which, args):
    assert _mutant(old, new, which, args) > 0, label


@pytest.mark.parametrize("n_tiles,num_kb,stages", [(1, 1, 3), (3, 16, 3), (4, 9, 6), (2, 20, 3), (5, 3, 2)])
def test_gemm_pipeline_protocol(n_tiles, num_kb, stages):
    """gemm_tc_kernel: TMA ring, slots released one k-block late under wgmma_wait<1>, K-chunk promotion."""
    from pipeline_protocol_model import gemm
    for seed in range(150):
        gemm(n_tiles, num_kb, seed, stages=stages).run()
