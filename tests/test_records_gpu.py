"""GPU: device-resident records (SURVEY 8(f) items 2 and 4): column extraction, survivor gather, the writers'
attribute transforms, and DataProcessor(device_records=True) == the host-gather mode, record for record."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def test_extract_gather_roundtrip(cuda, gsx_lib):
    import torch
    from gsx import records, synth
    a = synth.structured(50_000, "mixed")
    r = records.DeviceRecords.from_structured(a, cuda)
    xyz, op = r.xyz_opacity()
    assert np.array_equal(xyz.cpu().numpy(), np.column_stack((a["x"], a["y"], a["z"])))
    assert np.array_equal(op.cpu().numpy(), a["opacity"])
    idx = np.flatnonzero(np.random.default_rng(0).random(len(a)) < 0.37)
    g = r.gather(torch.from_numpy(idx.astype(np.int32)).to(cuda)).to_host()
    assert g.dtype == a.dtype and np.array_equal(g, a[idx])
    assert len(r.gather(torch.empty(0, dtype=torch.int32, device=cuda)).to_host()) == 0


def test_writer_transforms_match_numpy(cuda, gsx_lib):
    from gsx import records, synth
    a = synth.structured(200_000, "mixed")
    a["opacity"][:7] = [-200.0, 200.0, 0.0, -1e-9, 88.0, -88.0, 5.5]
    a["f_dc_0"][:4] = [-10.0, 10.0, 0.0, 1.7724539]
    r = records.DeviceRecords.from_structured(a, cuda)
    SH_C0 = 0.28209479177387814
    rgba = r.color_rgba8().cpu().numpy()
    for c, f in enumerate(("f_dc_0", "f_dc_1", "f_dc_2")):   # formats/splat.py:131-133 -- float32 ops only: bit-exact
        want = np.clip((0.5 + SH_C0 * a[f]) * 255, 0, 255).astype(np.uint8)
        assert np.array_equal(rgba[:, c], want), f
    want_a = np.clip((1.0 / (1.0 + np.exp(-a["opacity"]))) * 255, 0, 255).astype(np.uint8)   # splat.py:144
    assert np.array_equal(rgba[:, 3], want_a)
    rgba15 = r.color_rgba8(0.15).cpu().numpy()                      # spz.py:131 colour scale
    assert np.array_equal(rgba15[:, 1], np.clip((a["f_dc_1"] * 0.15 + 0.5) * 255.0, 0, 255).astype(np.uint8))
    sc = r.scale_exp().cpu().numpy()
    want_s = np.exp(np.column_stack((a["scale_0"], a["scale_1"], a["scale_2"])))
    assert np.array_equal(sc.view(np.uint32), want_s.view(np.uint32))


def test_dataprocessor_device_records_equals_host_gather(cuda, gsx_lib):
    from gsconverter.processing import DataProcessor
    from gsx import synth
    a = synth.structured(120_000, "mixed")
    outs = []
    for dev_rec in (False, True):
        dp = DataProcessor(a.copy())
        dp.device_records = dev_rec
        dp.defer_compaction = True
        dp.crop_by_bbox(-11, -11, -11, 11, 11, 11)
        dp.apply_alpha_filter(5)
        dp.apply_density_filter(1.0, 0.32, sensitivity=0.5, keep_multicluster=True)
        dp.remove_flyers(16, 2.0)
        outs.append(dp.data.copy())
    assert outs[0].dtype == outs[1].dtype and np.array_equal(outs[0], outs[1])
    assert 0 < len(outs[0]) < len(a)
