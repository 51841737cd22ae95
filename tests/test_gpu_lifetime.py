"""GPU: the runtime gives back the device memory it takes -- on shutdown, and when b200rt_init fails part-way.

b200rt_init allocates each replica's workspace in turn, then the root's staging buffers; a load adds its model's arenas on
every replica and, for some kinds, input slots.  Every one of these belongs to the runtime, so shutdown frees it all, and an
init that fails after the first replica frees what it had allocated (at wave_items=512 that is about 4 GB).  Free memory
comes from torch.cuda.mem_get_info(0); the baseline is taken after one whole init / shutdown cycle, so that loading the
library's modules is not counted, and the bar allows 1 GiB for other jobs on the card."""
import numpy as np
import pytest

import test_gpu_replica_kinds as RK
from oracle import bge_ref as R
from oracle import clip_ref as C

pytestmark = pytest.mark.gpu
MARGIN = 1 << 30
WAVE_ITEMS = 512


def _free():
    import torch

    return torch.cuda.mem_get_info(0)[0]


@pytest.fixture(scope="module")
def rt():
    import b200rt

    b200rt.shutdown()
    b200rt.init(devices=[0], wave_items=WAVE_ITEMS)
    b200rt.shutdown()
    yield b200rt
    b200rt.shutdown()


def _check_freed(baseline, what):
    lost = baseline - _free()
    print(f"{what}: {lost / 2**20:.0f} MiB below the baseline (bar {MARGIN / 2**20:.0f} MiB)")
    assert lost < MARGIN, f"{what} left {lost / 2**30:.2f} GiB allocated"


def _failed_init(rt):
    """init on device 0 and on a device that does not exist: replica 0 is allocated before the second is refused."""
    import torch

    with pytest.raises(rt.B200RTError) as e:
        rt.init(devices=[0, torch.cuda.device_count()], wave_items=WAVE_ITEMS)
    assert e.value.code == rt.E_INVALID, e.value


def _bge_base_embed(rt):
    g = R.BertGeometry(layers=2)
    flat = R.make_weights(g, 3, "trained")
    model = rt.EmbedModel(R.geometry_dict(g), R.pack_blob(flat, g))
    ids, lens = R.synth_ragged(5, 200, seed=5, min_len=3)
    return model.embed(ids, lens)


def test_failed_init_frees_its_memory(rt):
    baseline = _free()
    _failed_init(rt)
    _check_freed(baseline, "a failed init")


def test_init_after_a_failed_init_embeds_as_before(rt):
    rt.init(devices=[0])
    before = _bge_base_embed(rt)
    rt.shutdown()
    _failed_init(rt)
    rt.init(devices=[0])
    try:
        after = _bge_base_embed(rt)
    finally:
        rt.shutdown()
    assert np.array_equal(after.view(np.uint32), before.view(np.uint32))


def test_shutdown_frees_every_kind(rt):
    """A 2-layer model of each of the six kinds loaded and run once (CUDA graphs, classifier segment slots, ViT input slots
    and streams included), then shutdown."""
    baseline = _free()
    kinds, work = RK._kinds(), RK._workloads()
    rt.init(devices=[0], wave_items=WAVE_ITEMS)
    try:
        # kinds bert, bert_classifier, bert_splade, nomic_bert and clip_text; then vit
        for kind in ("bge_base", "classifier2", "splade", "nomic", "clip_text"):
            out = RK._call(kinds[kind][2](rt), work[kind]["one"])
            assert np.isfinite(out).all(), kind
        vg = C.VitGeometry(layers=2)
        vit = rt.ImageEmbedModel(C.geometry_dict(vg), C.pack_blob(C.make_weights(vg, 1, "trained"), vg))
        assert np.isfinite(vit.embed(C.synth_pixels(2, vg, 2))).all()
    finally:
        rt.shutdown()
    _check_freed(baseline, "shutdown")
