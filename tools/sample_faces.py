#!/usr/bin/env python
"""Random faces from FLAME parameters on the device: the counterpart of the reference's plots/generate_random_samples.py
on gif_b200.sampler.FlameSampler (eye-centred camera, condition render, EMA generator, image bytes; one CUDA graph per
batch).  Writes to --out:
    images.npy      uint8 (N, R, R, 3)      the generated faces
    conditions.npy  uint8 (2N, 256, 256, 3) texture renders (0..N-1) and normal maps (N..2N-1) fed to the generator
    mesh.npy        uint8 (N, 256, 256, 3)  the constant-albedo render the reference saves next to each sample
    params.npz      the reference's params_to_save: cam, shape, exp, pose, light_code (N,9,3), texture_code,
                    identity_indices (shape is stored once; the reference appends it twice, generate_random_samples.py:173-174)
Writing PNGs is left to the caller.

  python tools/sample_faces.py --out samples --n 64                                  # seeded weights, synthetic FLAME
  python tools/sample_faces.py --out samples --n 1000 --ckpt run/0.model --deca-rows deca.npy \\
      --flame-model generic_model.pkl --flame-lmk-embedding landmark_embedding.npy --tex-space FLAME_texture.npz

Parameters (generate_random_samples.py:100-121): shape[:3] and exp[:3] ~ N(0, 1), the rest 0; pose [0, U(-pi/8, pi/8), 0,
U(0, pi/12), 0, 0]; texture ~ N(0, 1); camera and light from the DECA rows of --deca-rows (row i mod their count), or from
``synthetic_deca_params``; identity indices ~ randint(vocab).  Without model files the synthetic FLAME-shaped model and
texture space stand in, as in GifTrainer.
"""
import argparse
import json
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from gif_b200.conditions import DECA_COLUMNS, DECA_SLICES  # noqa: E402

REFERENCE_VOCAB = 69158        # generate_random_samples.py:131 (the FFHQ identity embedding)


def draw_rows(n, seed, cam_lit_rows=None):
    """(n, 236) float32 DECA rows drawn as generate_random_samples.py:100-121 does, from one seeded numpy generator.
    cam_lit_rows: (M, >=236) rows whose camera and light columns row i takes (i mod M); None: ``synthetic_deca_params``."""
    rng = np.random.default_rng(seed)
    rows = np.zeros((n, DECA_COLUMNS), np.float32)
    col = lambda k: slice(*DECA_SLICES[k])
    rows[:, DECA_SLICES["shape"][0]:DECA_SLICES["shape"][0] + 3] = rng.normal(0, 1, (n, 3))
    rows[:, DECA_SLICES["exp"][0]:DECA_SLICES["exp"][0] + 3] = rng.normal(0, 1, (n, 3))
    pose = np.zeros((n, 6), np.float32)
    pose[:, 1] = rng.uniform(-np.pi / 8, np.pi / 8, n)
    pose[:, 3] = rng.uniform(0, np.pi / 12, n)
    rows[:, col("pose")] = pose
    rows[:, col("tex")] = rng.normal(0, 1, (n, DECA_SLICES["tex"][1] - DECA_SLICES["tex"][0]))
    if cam_lit_rows is None:
        from gif_b200.flame_synth import synthetic_deca_params
        cam_lit_rows = synthetic_deca_params(n, seed).numpy()
    src = np.asarray(cam_lit_rows, np.float32)[np.arange(n) % len(cam_lit_rows)]
    rows[:, col("cam")] = src[:, col("cam")]
    rows[:, col("lit")] = src[:, col("lit")]
    return rows


def draw_identities(n, vocab, seed):
    return np.random.default_rng(seed + 1).integers(0, vocab, n).astype(np.int64)


def params_to_save(rows, identities):
    """The dict generate_random_samples.py:146-147 fills (one entry per sample)."""
    s = lambda k: rows[:, slice(*DECA_SLICES[k])]
    return {"cam": s("cam"), "shape": s("shape"), "exp": s("exp"), "pose": s("pose"),
            "light_code": s("lit").reshape(-1, 9, 3), "texture_code": s("tex"), "identity_indices": identities}


def build_models(args, dev):
    """(FLAME, FLAMETex): from the model files when given, else the synthetic stand-ins GifTrainer uses."""
    from gif_b200.flame import FLAME, FLAMETex
    from gif_b200.flame_synth import synthetic_flame_model, synthetic_texture_space
    if args.flame_model:
        cfg = types.SimpleNamespace(flame_model_path=args.flame_model, flame_lmk_embedding_path=args.flame_lmk_embedding,
                                    shape_params=100, expression_params=50, tex_space_path=args.tex_space, tex_params=50)
        flame = FLAME(cfg)
    else:
        flame = FLAME.from_arrays(synthetic_flame_model())
    if args.tex_space:
        tex = FLAMETex(types.SimpleNamespace(tex_space_path=args.tex_space, tex_params=50))
    else:
        mean, basis = synthetic_texture_space(512, 50)
        tex = FLAMETex(mean=mean, basis=basis)
    return flame.to(dev), tex.to(dev)


def build_generator(args, dev):
    from gif_b200 import checkpoint
    from gif_b200.model.stg2_generator import StyledGenerator
    vocab = args.vocab
    ckpt = None
    if args.ckpt:
        ckpt = torch.load(args.ckpt, map_location="cpu", weights_only=True)
        emb = [v for k, v in ckpt["generator_running"].items() if k.endswith("image_embedding.embd_weight")]
        vocab = emb[0].shape[0] if emb else vocab
    torch.manual_seed(args.seed)
    G = StyledGenerator(embedding_vocab_size=vocab, rendered_flame_ascondition=True, normal_maps_as_cond=True,
                        core_tensor_res=4, w_truncation_factor=args.truncation, n_mlp=8)
    if ckpt is not None:
        checkpoint.load_reference_checkpoint(ckpt, g_running=G)
    return G.to(dev), vocab


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True)
    ap.add_argument("--n", type=int, default=64)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--resolution", type=int, default=256)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--precision", default="bf16x3", choices=("bf16x3", "tf32", "fp32"))
    ap.add_argument("--ckpt", help="reference-format checkpoint (generator_running is used); default: seeded weights")
    ap.add_argument("--vocab", type=int, default=REFERENCE_VOCAB, help="identity vocabulary of seeded weights")
    ap.add_argument("--truncation", type=float, default=1.0, help="w_truncation_factor")
    ap.add_argument("--deca-rows", help=".npy of DECA rows (M, >=236) to take cameras and lights from")
    ap.add_argument("--flame-model")
    ap.add_argument("--flame-lmk-embedding")
    ap.add_argument("--tex-space")
    ap.add_argument("--mesh-albedo", type=float, default=0.6,
                    help="constant albedo of mesh.npy (0..255 units; the reference's 0.6 renders black)")
    ap.add_argument("--no-eye-centering", action="store_true")
    ap.add_argument("--no-graphs", action="store_true")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("sample_faces needs a CUDA device")
    from gif_b200 import ops
    from gif_b200.conditions import DecaConditionRenderer
    from gif_b200.flame_synth import flame_uv
    from gif_b200.sampler import FlameSampler
    dev = torch.device("cuda:0")
    ops.set_precision(args.precision)
    flame, tex = build_models(args, dev)
    G, vocab = build_generator(args, dev)
    sampler = FlameSampler(G, DecaConditionRenderer(flame, tex, *flame_uv()), resolution=args.resolution,
                           batch_size=args.batch, eye_centering=not args.no_eye_centering, graphs=not args.no_graphs,
                           mesh_albedo=args.mesh_albedo)
    rows = draw_rows(args.n, args.seed, np.load(args.deca_rows) if args.deca_rows else None)
    ids = draw_identities(args.n, vocab, args.seed)
    out = sampler.sample(torch.from_numpy(rows).to(dev), torch.from_numpy(ids).to(dev))
    os.makedirs(args.out, exist_ok=True)
    for k in ("images", "conditions", "mesh"):
        np.save(os.path.join(args.out, f"{k}.npy"), out[k].cpu().numpy())
    np.savez(os.path.join(args.out, "params.npz"), **params_to_save(out["rows"].cpu().numpy(), ids))
    print(json.dumps({"n": args.n, "resolution": args.resolution, "vocab": vocab, "precision": args.precision,
                      "nan_cameras": int(torch.isnan(out["cam"]).any(1).sum()), "out": args.out}))


if __name__ == "__main__":
    main()
