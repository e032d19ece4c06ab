"""Generate tests/golden/scans/* from the REAL reference's Tanks and BlendedMVS dataset classes
(/root/reference/datasets), run in the build container.  TEST INFRASTRUCTURE.

    python oracle/make_golden_scans.py

Writes a small seeded fixture in both layouts (casmvsnet_pl_b200.synth_scenes) under
tests/golden/scans/{tanks,blendedmvs}/ and records what TanksDataset / BlendedMVSDataset derive
from it in test mode (metas, proj_mats, scale_factors and every __getitem__: imgs, proj_mats,
init_depth_min, depth_interval) into tests/golden/scans/{tanks,blendedmvs}.npz.
"""
import os
import shutil
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("CASMVS_REFERENCE_ROOT", "/root/reference")
OUT = os.path.join(ROOT, "tests", "golden", "scans")
sys.path.insert(0, ROOT)

# fixture parameters, shared with tests/test_scan_ingest.py through the npz
TANKS = dict(split="intermediate", scan="Family", n_views=5, image_wh=(80, 48), img_wh=(64, 32),
             reader_views=3)
BMVS = dict(scan="5a3ca9cb270f0e3f14d0eddb", n_views=6, image_wh=(96, 72), img_wh=(64, 64),
            reader_views=3, n_depths_arg=2.65)


def _record(ds, scan_of):
    out = {"metas": np.array([[m[2]] + m[3] + [-1] * (8 - len(m[3])) for m in ds.metas]),
           "imgs": [], "proj_mats": [], "init_depth_min": [], "depth_interval": [], "ref": []}
    for i in range(len(ds)):
        s = ds[i]
        out["imgs"].append(s["imgs"].numpy())
        out["proj_mats"].append(s["proj_mats"].numpy())
        out["init_depth_min"].append(s["init_depth_min"].item())
        out["depth_interval"].append(s["depth_interval"].item())
        out["ref"].append(s["scan_vid"][1])
    out = {k: np.array(v) for k, v in out.items()}
    pm = ds.proj_mats[scan_of]
    out["view_ids"] = np.array(sorted(pm))
    out["view_proj"] = torch.stack([pm[v][0] for v in sorted(pm)]).numpy()
    out["view_depth_min"] = np.array([pm[v][1] for v in sorted(pm)])
    return out


def main():
    from casmvsnet_pl_b200 import synth_scenes
    shutil.rmtree(OUT, ignore_errors=True)
    os.makedirs(OUT)
    sys.path.insert(0, REF)
    from datasets.blendedmvs import BlendedMVSDataset   # noqa: E402
    from datasets.tanks import TanksDataset             # noqa: E402

    t = TANKS
    synth_scenes.make_tanks(os.path.join(OUT, "tanks"), t["split"], t["scan"], t["n_views"],
                            t["image_wh"], seed=1)
    # TanksDataset opens the pair.txt of every scan of the split (tanks.py:67-74): run it on a
    # copy of the fixture in which the other scans have empty pair files
    import tempfile
    tmp = tempfile.mkdtemp()
    shutil.copytree(os.path.join(OUT, "tanks"), os.path.join(tmp, "tanks"))
    from casmvsnet_pl_b200.eval_pipeline import TanksTestScan
    for other in TanksTestScan.SCANS[t["split"]]:
        if other != t["scan"]:
            os.makedirs(os.path.join(tmp, "tanks", t["split"], other))
            with open(os.path.join(tmp, "tanks", t["split"], other, "pair.txt"), "w") as f:
                f.write("0\n")
    ds = TanksDataset(os.path.join(tmp, "tanks"), t["split"], n_views=t["reader_views"],
                      img_wh=t["img_wh"])
    rec = _record(ds, t["scan"])
    rec.update(img_wh=np.array(t["img_wh"]), n_views=t["reader_views"])
    np.savez_compressed(os.path.join(OUT, "tanks.npz"), **rec)
    shutil.rmtree(tmp)

    b = BMVS
    root = synth_scenes.make_blendedmvs(os.path.join(OUT, "blendedmvs"), b["scan"], b["n_views"],
                                        b["image_wh"], seed=2, n_few=3, lists=("val",))
    ds = BlendedMVSDataset(root, "val", n_views=b["reader_views"], depth_interval=b["n_depths_arg"],
                           img_wh=b["img_wh"])
    rec = _record(ds, b["scan"])
    rec.update(img_wh=np.array(b["img_wh"]), n_views=b["reader_views"],
               n_depths_arg=b["n_depths_arg"], scale_factor=ds.scale_factors[b["scan"]])
    np.savez_compressed(os.path.join(OUT, "blendedmvs.npz"), **rec)
    print("wrote", sorted(os.listdir(OUT)))


if __name__ == "__main__":
    main()
