"""CPU tests of the host side: the C-ABI library loads and exports every declared symbol, the product path
refuses to run without CUDA (no CPU fallback), RoPE tables are bit-identical to the oracle, and parameter names match
the reference's (stored golden data)."""
import os
import re
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def test_cabi_exports_every_declared_symbol():
    from scail_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "scail_b200.h")).read()
    declared = set(re.findall(r"^(?:int|const char\*)\s+(scail_\w+)\s*\(", hdr, flags=re.M))
    assert len(declared) >= 18
    h = _lib.lib()
    for name in declared:
        assert hasattr(h, name), name
    assert declared - {"scail_last_error"} == set(_lib.SIGNATURES), declared ^ set(_lib.SIGNATURES)
    assert h.scail_version() == 100


def test_no_cpu_fallback():
    from scail_b200 import ops
    from scail_b200.dit import DiffusionTransformer
    from scail_b200.wan_vae import WanVAE
    with pytest.raises(RuntimeError):
        ops.gemm(torch.zeros(8, 8, dtype=torch.bfloat16), torch.zeros(8, 8, dtype=torch.bfloat16))
    m = DiffusionTransformer(hidden_size=256, num_attention_heads=2, inner_hidden_size=512, num_layers=1, text_dim=64,
                             time_embed_dim=256)
    with pytest.raises(RuntimeError):
        m(torch.zeros(1, 2, 16, 8, 8), timesteps=torch.zeros(1), context=torch.zeros(1, 4, 64),
          ref_concat=torch.zeros(1, 1, 16, 8, 8), concat_smpl_render=torch.zeros(1, 2, 16, 4, 4),
          image_clip_features=torch.zeros(1, 257, 1280))
    v = WanVAE(dim=16, device="cpu")
    with pytest.raises(RuntimeError):
        v.decode([torch.zeros(16, 1, 4, 4)])
    if not torch.cuda.is_available():  # without a device the library itself reports the failure
        from scail_b200 import _lib
        assert _lib.lib().scail_device_sm_count(0) < 0
        assert b"CUDA" in _lib.lib().scail_last_error()


def test_product_does_not_import_oracle():
    for dirpath, _, files in os.walk(os.path.join(ROOT, "scail_b200")):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dirpath, f)).read()
                assert "import oracle" not in src and "from oracle" not in src, f
                assert "import baseline" not in src and "from baseline" not in src, f  # the library-path arm is bench-only


def test_rope_tables_bit_identical_to_oracle():
    from oracle import dit_oracle as O
    from scail_b200 import rope
    # the token grids of 512x512, 512x896 (landscape and portrait) and 480x832 latents
    for (T, H, W) in [(3, 4, 6), (4, 8, 8), (21, 32, 32), (21, 32, 56), (21, 56, 32), (21, 30, 52)]:
        c, s = rope.build_tables_cpu(128, T, H, W)
        c2, s2 = O.rope_tables(128, T, H, W, 21, 150, 150)
        assert torch.equal(c, c2) and torch.equal(s, s2)
    c, s = rope.build_tables_cpu(128, 2, 4, 4, 2, 4)  # SP-style shifts (dit_video_crossattn_sc_xc.py:1578-1585)
    c2, s2 = O.rope_tables(128, 2, 4, 4, 21, 150, 150, h_shift=2, w_shift=4)
    assert torch.equal(c, c2) and torch.equal(s, s2)


# the pre-chunked context-parallel forms the CP launch-shape test runs: (token grid T, H, W of the latent, chunk_dim, P).
# 512x896 -> 21x32x56, 480x832 -> 21x30x52; chunk_dim 3 at 480x832 would leave a 15-row pose latent per rank, which does
# not patchify
CHUNK_CASES = [((21, 32, 56), 3, 2), ((21, 32, 56), 3, 4), ((21, 32, 56), 4, 2), ((21, 32, 56), 4, 4), ((21, 30, 52), 4, 2)]


def chunk_shifts(T, H, W, chunk_dim, P, p):
    """(rope_H, rope_W, rope_H_shift, rope_W_shift) of rank p when the latents are chunked on H (chunk_dim 3) or W (4)."""
    if chunk_dim == 3:
        return H // P, W, p * (H // P), 0
    return H, W // P, 0, p * (W // P)


def chunk_tokens(T, H, W, chunk_dim, P, p):
    """The global token indices (into the one-GPU ref || noise || pose sequence of a T x H x W token grid) of rank p's
    local sequence when the latent, the reference and the pose are each chunked on H (chunk_dim 3) or W (4) into P parts,
    in local order."""
    def part(t, h, w, base):
        idx = torch.arange(t * h * w).view(t, h, w) + base
        return (idx[:, p * h // P:(p + 1) * h // P] if chunk_dim == 3 else idx[:, :, p * w // P:(p + 1) * w // P]).reshape(-1)
    n_ref, n_seq = H * W, T * H * W
    return torch.cat([part(1, H, W, 0), part(T, H, W, n_ref), part(T, H // 2, W // 2, n_ref + n_seq)])


def test_shifted_rope_tables_at_production_chunks_bit_identical_to_oracle():
    from oracle import dit_oracle as O
    from scail_b200 import rope
    for (T, H, W), cd, P in CHUNK_CASES:
        for p in range(P):
            h, w, hs, ws = chunk_shifts(T, H, W, cd, P, p)
            c, s = rope.build_tables_cpu(128, T, h, w, hs, ws)
            c2, s2 = O.rope_tables(128, T, h, w, 21, 150, 150, h_shift=hs, w_shift=ws)
            assert torch.equal(c, c2) and torch.equal(s, s2), ((T, H, W), cd, P, p)


def test_each_ranks_shifted_tables_are_the_one_gpu_rows_of_its_tokens():
    """Rank p's shifted tables equal the one-GPU tables at chunk_tokens(p), bit for bit.  Every shift here is even, so the 2x2
    average pooling of the pose rows pairs the same grid rows and columns locally as on one GPU (an odd shift would pool
    across the pairs and give other values)."""
    from scail_b200 import rope
    for (T, H, W), cd, P in CHUNK_CASES:
        c, s = rope.build_tables_cpu(128, T, H, W)
        for p in range(P):
            h, w, hs, ws = chunk_shifts(T, H, W, cd, P, p)
            assert hs % 2 == 0 and ws % 2 == 0
            idx = chunk_tokens(T, H, W, cd, P, p)
            assert idx.numel() * P == c.shape[0]
            cl, sl = rope.build_tables_cpu(128, T, h, w, hs, ws)
            assert torch.equal(cl, c[idx]) and torch.equal(sl, s[idx]), ((T, H, W), cd, P, p)
    # the ranks' tokens partition the sequence
    for (T, H, W), cd, P in CHUNK_CASES:
        allidx = torch.cat([chunk_tokens(T, H, W, cd, P, p) for p in range(P)])
        assert torch.equal(allidx.sort().values, torch.arange(allidx.numel()))


def test_state_dict_names_match_reference_golden():
    from scail_b200.dit import DiffusionTransformer
    from scail_b200.wan_vae import WanVAE
    g = torch.load(os.path.join(GOLD, "dit_c1.pt"))
    cfg = g["cfg"]
    m = DiffusionTransformer(hidden_size=cfg["hidden"], num_attention_heads=cfg["heads"], inner_hidden_size=cfg["inner"],
                             num_layers=cfg["layers"], text_dim=cfg["text_dim"], time_embed_dim=cfg["hidden"])
    ours = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    ref = {k: tuple(v.shape) for k, v in g["state_dict"].items()}
    assert ours == ref
    gv = torch.load(os.path.join(GOLD, "vae_small.pt"))
    v = WanVAE(dim=gv["dim"], device="cpu")
    ours = {k: tuple(t.shape) for k, t in v.model.state_dict().items()}
    ge = torch.load(os.path.join(GOLD, "vae_encode_small.pt"))
    ref = {k: tuple(t.shape) for k, t in gv["state_dict"].items()}
    ref.update({k: tuple(t.shape) for k, t in ge["state_dict"].items()})
    assert ours == ref  # decoder.* + conv2.* (decode) and encoder.* + conv1.* (encode): the whole Wan2.1_VAE.pth layout


def test_sampler_schedule_matches_golden():
    from scail_b200 import sampler
    s = torch.load(os.path.join(GOLD, "sampler.pt"))
    assert torch.equal(sampler.make_flow_timesteps(50, 5.0), s["sigmas"])


def test_bench_flop_model():
    sys.path.insert(0, ROOT)
    import bench
    assert bench.seq_len() == 27904
    assert abs(bench.block_flops(27904) / 1e12 - 33.144) < 0.01          # BASELINE.md table
    assert abs(bench.forward_flops(27904) / 1e12 - 1325.8) < 0.1


def test_bench_reference_arm_json_contract():
    """`bench.py --impl reference` (the CPU arm: oracle port on the host cores, bounded sample) prints one JSON line with
    the contract's keys.  Uses a reduced sample so the CPU suite stays short."""
    import json
    import subprocess
    code = ("import sys, json; sys.argv=['bench.py','--impl','reference','--steps','1','--warmup','0'];"
            "import bench; bench.CPU_ARM_BUDGET_S=0.0; bench.main()")  # budget 0 -> the reduced 9x32x32 sample
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    line = [l for l in r.stdout.splitlines() if l.startswith("{")][-1]
    d = json.loads(line)
    assert d["impl"] == "reference" and d["unit"] == "steps/s" and d["higher_is_better"] is True
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1 and "sample" in d["cpu_baseline"]
    assert d["e2e"] == {"value": d["value"], "unit": "steps/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert d["value"] > 0 and d["config"]["seq_len"] == 27904


def test_sample_long_matches_reference_golden():
    """RFSamplerLong (sampling.py:986-1085) host logic vs the golden produced by the UNMODIFIED reference sampler driving a
    deterministic stand-in network (tests/golden/gen_sampler_long.py): tile scheduling, triangular blend, CFG (incl. the uncond
    padding rule of guiders.py:52-53), Euler update, flow schedule."""
    import sys
    from scail_b200 import sampler
    gdir = os.path.join(os.path.dirname(__file__), "golden")
    sys.path.insert(0, gdir)
    from fake_network import fake_network
    g = torch.load(os.path.join(gdir, "sampler_long.pt"))

    def denoise(x_tile, sigma, c_k, u_k):  # VanillaCFG.prepare_inputs + __call__ around the stand-in network
        ctx = sampler.prepare_context(c_k, u_k)
        both = dict(crossattn=ctx, concat_smpl_render=c_k["concat_smpl_render"])
        v = fake_network(torch.cat([x_tile] * 2), torch.cat([sigma.view(1) * 1000.0] * 2), both)
        vu, vc = v.chunk(2)
        return vu + g["scale"] * (vc - vu)

    out = sampler.sample_long(None, g["x"].clone(), g["cond"], g["uc"], g["tile_indices"], num_steps=g["num_steps"],
                              shift_scale=g["shift_scale"], scale=g["scale"], denoise=denoise)
    assert out.shape == g["out"].shape
    assert torch.allclose(out, g["out"], rtol=0, atol=2e-6), float((out - g["out"]).abs().max())
    assert sampler.make_tile_indices(13, 5, 4) == g["tile_indices"]


def test_checkpoint_layout_roundtrip_and_error_behaviour(tmp_path):
    """SAT checkpoint layout (sat/training/model_io.py:36-48, 233-356): latest -> <iter>/mp_rank_00_model_states.pt ->
    sd['module'] with the engine prefix; missing keys raise unless force_inference, unexpected keys only warn."""
    import pytest
    from scail_b200 import checkpoint as C
    from scail_b200.dit import DiffusionTransformer
    cfg = dict(hidden_size=256, num_attention_heads=2, inner_hidden_size=512, num_layers=1, text_dim=64, time_embed_dim=256)
    torch.manual_seed(0)
    a = DiffusionTransformer(**cfg)
    C.save_checkpoint(a, str(tmp_path), 1000)
    assert open(tmp_path / "latest").read() == "1000" and (tmp_path / "1000" / "mp_rank_00_model_states.pt").is_file()
    torch.manual_seed(1)
    b = DiffusionTransformer(**cfg)
    assert C.load_checkpoint(b, str(tmp_path)) == 1000 and not b.training
    for (k, va), (_, vb) in zip(a.state_dict().items(), b.state_dict().items()):
        assert torch.equal(va, vb), k
    # a checkpoint that lacks a parameter: inference refuses unless forced (model_io.py:303-307)
    sd = torch.load(tmp_path / "1000" / "mp_rank_00_model_states.pt")
    del sd["module"][C.DIT_PREFIX + "mixins.final_layer.linear.bias"]
    sd["module"][C.DIT_PREFIX + "not_a_parameter"] = torch.zeros(1)
    sd["module"]["conditioner.something"] = torch.zeros(1)  # other engine sub-modules are filtered out by the prefix
    torch.save(sd, tmp_path / "1000" / "mp_rank_00_model_states.pt")
    with pytest.warns(UserWarning, match="unexpected_keys"), pytest.raises(ValueError, match="Missing keys for inference"):
        C.load_checkpoint(b, str(tmp_path))
    with pytest.warns(UserWarning):
        assert C.load_checkpoint(b, str(tmp_path), force_inference=True) == 1000
    (tmp_path / "latest").write_text("garbage")
    with pytest.raises(ValueError, match="Invalid metadata"):
        C.load_checkpoint(b, str(tmp_path))
    (tmp_path / "latest").write_text("release")
    assert C.get_checkpoint_name(str(tmp_path), *C.get_checkpoint_iteration(str(tmp_path))).endswith("release/mp_rank_00_model_states.pt")
