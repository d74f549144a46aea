"""TEST INFRASTRUCTURE ONLY -- writes ``tests/golden/fid_inception.npz``: the UNMODIFIED reference FID network
(my_utils/pytorch_fid/inception.py InceptionV3, imported from the reference tree the way ``oracle/ref_import.py`` imports
the reference) evaluated in float64 on the CPU with seeded weights, and the agreement of the in-repo oracle
(``oracle/inception_oracle.py``) with it in ``tests/golden/FID_ORACLE_VS_REFERENCE.txt``.

  * Weights: ``inception_oracle.seeded_state_dict(SEED)``.  The reference module fetches its weights with
    ``load_state_dict_from_url``; before the module is imported the torch hub loaders are replaced by a function that raises,
    and after the import the module's own name is pointed at the seeded state dict -- the recipe never reaches the network.
  * BatchNorm running statistics: calibrated once on a seeded batch (train-mode pass, momentum=None) so that every layer
    stays O(1); they are stored (small).  Conv weights are regenerated from the seed and their sha256 is stored.
  * Inputs: 2 images at 299^2, 2 at 256^2 (resize path), 2 at 256^2 with resize_input=False.
  * Stored: block 3 in full, seeded samples of blocks 0-2 (``golden_util.sample``), the reference's own float32 error.

Run where the reference tree and torchvision exist (a few minutes on 8 cores):   python tools/make_fid_golden.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import golden_util as gu  # noqa: E402
from oracle import inception_oracle as IO  # noqa: E402
from oracle import ref_import  # noqa: E402

SEED = 2015


# reference module names (blocks.i.j, as InceptionV3.__init__ builds them, inception.py:85-125) -> torchvision names
PREFIX = {"blocks.0.0": "Conv2d_1a_3x3", "blocks.0.1": "Conv2d_2a_3x3", "blocks.0.2": "Conv2d_2b_3x3",
          "blocks.1.0": "Conv2d_3b_1x1", "blocks.1.1": "Conv2d_4a_3x3"}
PREFIX.update({f"blocks.2.{i}": n for i, n in enumerate(["Mixed_5b", "Mixed_5c", "Mixed_5d", "Mixed_6a", "Mixed_6b",
                                                         "Mixed_6c", "Mixed_6d", "Mixed_6e"])})
PREFIX.update({f"blocks.3.{i}": n for i, n in enumerate(["Mixed_7a", "Mixed_7b", "Mixed_7c"])})


def _as_blocks(sd):
    inv = {v: k for k, v in PREFIX.items()}
    out = {}
    for k, v in sd.items():
        if k.startswith("fc."):
            continue
        head = k.split(".")[0]
        out[inv[head] + k[len(head):]] = v
    return out


def _no_download(*a, **k):
    raise RuntimeError("make_fid_golden: the reference tried to download weights; the recipe must never reach the network")


def load_reference_fid_module():
    import torch.hub
    import torch.utils.model_zoo
    torch.hub.load_state_dict_from_url = _no_download
    torch.utils.model_zoo.load_url = _no_download
    if ref_import.REF_ROOT not in sys.path:
        sys.path.insert(0, ref_import.REF_ROOT)
    import my_utils.pytorch_fid.inception as ref_inception
    if ref_inception.load_state_dict_from_url is not _no_download:
        raise RuntimeError("reference inception.py bound a weight loader the recipe did not intercept")
    return ref_inception


def rel_l2(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


def main():
    torch.set_num_threads(os.cpu_count() or 8)
    ref = load_reference_fid_module()
    sd = IO.seeded_state_dict(SEED)
    ref.load_state_dict_from_url = lambda *a, **k: sd
    with ref_import.quiet():
        model = ref.InceptionV3(output_blocks=[0, 1, 2, 3], resize_input=True, normalize_input=True)
    model = model.double()
    model.load_state_dict(_as_blocks(sd))   # the float64 values, not their float32 copy
    # BN calibration: one train-mode pass with cumulative statistics
    bns = [m for m in model.modules() if isinstance(m, torch.nn.BatchNorm2d)]
    for m in bns:
        m.reset_running_stats()
        m.momentum = None
    model.train()
    calib = torch.from_numpy(np.random.Generator(np.random.PCG64(30)).uniform(0.0, 1.0, (4, 3, 299, 299)))
    with torch.no_grad():
        model(calib)
    model.eval()
    out = {"seed": np.int64(SEED), "weights_sha256": np.array(IO.weights_sha256(sd))}
    msd = model.state_dict()
    for k, v in msd.items():
        if k.endswith(".bn.running_mean") or k.endswith(".bn.running_var"):
            head = ".".join(k.split(".")[:3])
            name = PREFIX[head] + k[len(head):-len(".bn.running_mean" if k.endswith("mean") else ".bn.running_var")]
            out[("bn_mean/" if k.endswith("mean") else "bn_var/") + name] = v.numpy().copy()
    missing = [n for n, *_ in IO.CONVS if f"bn_mean/{n}" not in out]
    assert not missing, missing
    g_sd = IO.golden_state_dict(out)
    report = []
    model32 = None
    for case, x, resize in IO.golden_inputs(out):
        model.resize_input = resize
        with torch.no_grad():
            ref_out = model(x)
            orc = IO.forward(g_sd, x, (0, 1, 2, 3), resize_input=resize)
        for i, (a, b) in enumerate(zip(orc, ref_out)):
            e = rel_l2(a.numpy(), b.numpy())
            report.append((f"{case} block {i} (shape {tuple(b.shape)})", e))
            assert e < 1e-12, (case, i, e)
            if i == 3:
                out[f"{case}_b3"] = b.reshape(b.shape[0], -1).numpy()
            else:
                out[f"{case}_b{i}"], out[f"{case}_b{i}_sum"] = gu.sample(b, 4096, 40 + i)
                out[f"{case}_b{i}_shape"] = np.array(b.shape)
        if model32 is None:
            import copy
            model32 = copy.deepcopy(model).float()
        model32.resize_input = resize
        with torch.no_grad():
            r32 = model32(x.float())[3]
        out[f"{case}_ref32_err"] = rel_l2(r32.double().numpy(), ref_out[3].numpy())
        print(case, "done", flush=True)
    np.savez_compressed(os.path.join(gu.GOLDEN_DIR, "fid_inception.npz"), **{k: np.asarray(v) for k, v in out.items()})
    w = max(len(n) for n, _ in report)
    with open(os.path.join(gu.GOLDEN_DIR, "FID_ORACLE_VS_REFERENCE.txt"), "w") as f:
        f.write("# oracle/inception_oracle.py vs the unmodified reference InceptionV3 (my_utils/pytorch_fid/inception.py), float64, "
                "relative L2 error; written by tools/make_fid_golden.py\n")
        f.write("# reference float32 vs float64, block 3: " +
                ", ".join(f"{c} {out[f'{c}_ref32_err']:.3e}" for c, _, _ in IO.golden_inputs(out)) + "\n")
        for n, e in report:
            f.write(f"{n:<{w}}  {e:.3e}\n")
    print("written", os.path.join(gu.GOLDEN_DIR, "fid_inception.npz"))


if __name__ == "__main__":
    main()
