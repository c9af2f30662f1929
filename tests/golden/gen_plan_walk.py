"""Writes tests/golden/plan_walk.jsonl: what the weight-key spec, the FLOP count, the K/V exchange size and the launch
and module lists return over a grid of configs and latent shapes.  tests/test_plan.py asserts that they still return
exactly this, so a change to the UNet walk that moves any of them shows.

    python tests/golden/gen_plan_walk.py
"""
import dataclasses
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from diffuman4d_b200.config import UNetConfig  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "plan_walk.jsonl")
SHAPES = [(16, 64, 64), (24, 64, 64), (16, 128, 128), (4, 32, 32), (3, 16, 16), (2, 24, 24)]   # (F, h, w); B = 2F


def configs():
    """name -> UNetConfig: four base layouts, each also with one knob of the walk changed."""
    attn2 = UNetConfig.tiny(cross_attention_dim=(64, 128, 256, 256), use_linear_projection=False,
                            enable_pose_encoder=False, enable_tem_embeds=False, in_channels=15)
    out = {}
    for base, cfg in (("sd21", UNetConfig.sd21()), ("ctor_default", UNetConfig.ctor_default()),
                      ("tiny", UNetConfig.tiny()), ("tiny_attn2", attn2)):
        out[base] = cfg
        for n3d in range(5):
            out[f"{base}-n3d{n3d}"] = dataclasses.replace(cfg, num_3d_attn_blocks=n3d)
        for L in (1, 2, 3):
            out[f"{base}-L{L}"] = dataclasses.replace(cfg, layers_per_block=L)
        out[f"{base}-pose{int(not cfg.enable_pose_encoder)}"] = dataclasses.replace(
            cfg, enable_pose_encoder=not cfg.enable_pose_encoder)
        out[f"{base}-tem{int(not cfg.enable_tem_embeds)}"] = dataclasses.replace(
            cfg, enable_tem_embeds=not cfg.enable_tem_embeds)
        out[f"{base}-linproj{int(not cfg.use_linear_projection)}"] = dataclasses.replace(
            cfg, use_linear_projection=not cfg.use_linear_projection)
    out["tiny-L3-n3d4-attn2"] = dataclasses.replace(attn2, layers_per_block=3, num_3d_attn_blocks=4,
                                                    enable_pose_encoder=True, enable_tem_embeds=True)
    return out


def sha(obj):
    return hashlib.sha256(json.dumps(obj).encode()).hexdigest()


def generate():
    from diffuman4d_b200.flops import unet_flops
    from diffuman4d_b200.sharded import exchange_bytes
    from diffuman4d_b200.weights import state_dict_spec
    from gemm_shapes import plan_shapes
    from test_gpu_attention_fp64 import PLANS, SHARDED, attention_launches
    from test_gpu_unet_modules import module_plan

    def launches(d):
        return sorted([list(k), n] for k, n in d.items())

    out = {"state_dict_spec": {}, "module_plan": {}, "unet_flops": {}, "exchange_bytes": {}, "attention_launches": {},
           "plan_shapes": {}}
    for name, cfg in configs().items():
        out["state_dict_spec"][name] = sha([[k, list(v)] for k, v in state_dict_spec(cfg).items()])
        out["module_plan"][name] = {F: sha(module_plan(cfg, F)) for F in (1, 4)}
        out["unet_flops"][name] = {f"{F}@{h}x{w}": unet_flops(cfg, 2 * F, F, h, w) for F, h, w in SHAPES}
    for name in ("tiny", "sd21", "ctor_default"):
        for n3d in range(5):
            cfg = dataclasses.replace(getattr(UNetConfig, name)(), num_3d_attn_blocks=n3d)
            out["exchange_bytes"][f"{name}-n3d{n3d}"] = {
                f"{F}@{lat}": exchange_bytes(cfg, F, lat, lat) for F in (2, 4, 16, 24) for lat in (16, 24, 64, 128)}
    for name, (cfg, F, h, w) in PLANS.items():
        out["attention_launches"][name] = launches(attention_launches(cfg, F, h, w))
    for name, (cfg, F, h, w, r) in SHARDED.items():
        out["attention_launches"][name] = launches(attention_launches(cfg, F, h, w, ranks=r))
    for plan, (B, s0) in {"W16@64": (32, 64), "W24@64": (48, 64), "W16@128": (32, 128)}.items():
        out["plan_shapes"][plan] = [[kind, nm, cnt, {k: (list(v) if isinstance(v, tuple) else v) for k, v in spec.items()}]
                                    for kind, nm, cnt, spec in plan_shapes(B, s0)]
    return out


def read(path=OUT):
    """The fixture as generate() returns it after a JSON round trip: {table: {key: value}}."""
    out = {}
    with open(path) as fh:
        for line in fh:
            table, key, value = json.loads(line)
            out.setdefault(table, {})[key] = value
    return out


if __name__ == "__main__":
    with open(OUT, "w") as fh:   # one line per table entry
        for table, rows in sorted(json.loads(json.dumps(generate())).items()):
            for key, value in sorted(rows.items()):
                fh.write(json.dumps([table, key, value], sort_keys=True) + "\n")
    print(f"wrote {OUT}")
