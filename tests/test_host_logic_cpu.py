"""CPU tests of the host-side logic: weight packing, tile-box heuristics, module structure / state-dict
compatibility with the reference layout (Appendix B of SURVEY.md), timestep forms, router merge indexing."""
import math

import pytest
import torch

from ctrl_adapter_b200 import adapter as A
from ctrl_adapter_b200 import ops
from oracle import cases


def test_choose_box_covers_and_products():
    for (w, h, n) in [(128, 128, 16), (64, 64, 2), (8, 8, 3), (16, 9, 2), (128, 72, 56), (1, 1, 5), (4, 4, 1)]:
        bw, bh, bn = ops.choose_box(w, h, n)
        assert bw * bh * bn == 128
        tiles = math.ceil(w / bw) * math.ceil(h / bh) * math.ceil(n / bn)
        assert tiles * 128 >= w * h * n
    assert ops.choose_box(8, 8, 16) == (8, 8, 2)       # two 8x8 samples per tile, no padding
    assert ops.choose_box(128, 128, 1)[0] == 128


def test_pack_conv_weight_layout():
    w = torch.arange(2 * 3 * 3 * 3, dtype=torch.float32).reshape(2, 3, 3, 3)
    p = ops.pack_conv_weight(w, 8).float()
    assert p.shape == (2, 9 * 8)
    # tap (dy, dx) = (1, 2) -> index 5; channel 2
    assert p[1, 5 * 8 + 2] == w[1, 2, 1, 2]
    assert float(p[:, 3:8].abs().max()) == 0.0  # zero padded channels
    w3 = torch.randn(4, 8, 3, 1, 1)
    p3 = ops.pack_conv_weight(w3).float()
    assert torch.equal(p3[:, 8:16], w3[:, :, 1, 0, 0].to(torch.bfloat16).float())


def test_pack_geglu_interleave():
    d, k = 512, 16
    w = torch.randn(2 * d, k)
    b = torch.randn(2 * d)
    wi, bi = ops.pack_geglu_weight(w, b, 256)
    # tile t holds value rows [128t, 128t+128) then gate rows [d+128t, d+128t+128)
    assert torch.equal(wi[256:384], w[128:256]) and torch.equal(wi[384:512], w[d + 128:d + 256])
    assert torch.equal(bi[0:128], b[0:128]) and torch.equal(bi[128:256], b[d:d + 128])


@pytest.mark.parametrize("kw,okind", [(cases.ADAPTER_SDXL_KW, "sdxl"), (cases.ADAPTER_VIDEO_KW, "video")])
def test_adapter_state_dict_matches_reference_layout(kw, okind):
    from oracle.adapter import ControlNetAdapter as O
    with torch.device("meta"):
        ours, ref = A.ControlNetAdapter(**kw), O(**kw)
    a, b = ours.state_dict(), ref.state_dict()
    assert set(a) == set(b)
    assert all(a[k].shape == b[k].shape for k in a)
    assert ours.get_down_block_ids() == ref.get_down_block_ids()
    assert ours.get_down_block_channels() == ref.get_down_block_channels()


def test_controlnet_and_unet_state_dicts_match_reference_layout():
    from ctrl_adapter_b200.controlnet import ControlNetModel
    from ctrl_adapter_b200.unet_sdxl import UNet2DConditionModel
    from oracle.controlnet import ControlNetModel as OCN
    from oracle.unet_sdxl import UNet2DConditionModel as OU
    with torch.device("meta"):
        for ours, ref in ((ControlNetModel(**cases.CONTROLNET_KW), OCN(**cases.CONTROLNET_KW)),
                          (UNet2DConditionModel(), OU())):
            a, b = ours.state_dict(), ref.state_dict()
            assert set(a) == set(b), (sorted(set(a) - set(b))[:5], sorted(set(b) - set(a))[:5])
            assert all(a[k].shape == b[k].shape for k in a)


def test_video_unet_state_dicts_match_reference_layout():
    """I2VGen-XL and SVD UNets: same keys / shapes as the (oracle restatement of the) reference classes, and the published
    parameter count of the SVD UNet (1 524 623 082 for stable-video-diffusion-img2vid)."""
    from ctrl_adapter_b200.unet_i2vgen import I2VGenXLUNet
    from ctrl_adapter_b200.unet_svd import UNetSpatioTemporalConditionModel
    from oracle.unet_i2vgen import I2VGenXLUNet as OI
    from oracle.unet_svd import UNetSpatioTemporalConditionModel as OS
    with torch.device("meta"):
        for ours, ref in ((I2VGenXLUNet(), OI()),
                          (UNetSpatioTemporalConditionModel(**cases.UNET_SVD_KW), OS(**cases.UNET_SVD_KW))):
            a, b = ours.state_dict(), ref.state_dict()
            assert set(a) == set(b), (sorted(set(a) - set(b))[:5], sorted(set(b) - set(a))[:5])
            assert all(a[k].shape == b[k].shape for k in a), [k for k in a if a[k].shape != b[k].shape][:5]
        n_svd = sum(p.numel() for p in ref.parameters())
    assert n_svd == 1_524_623_082


def test_svd_unet_rejects_unsupported_topologies():
    from ctrl_adapter_b200.unet_svd import UNetSpatioTemporalConditionModel
    with torch.device("meta"):
        with pytest.raises(ValueError):
            UNetSpatioTemporalConditionModel(down_block_types=("DownBlockSpatioTemporal",) * 3)
        with pytest.raises(NotImplementedError):
            UNetSpatioTemporalConditionModel(block_out_channels=(64, 128, 256, 256), num_attention_heads=(1, 2, 4, 4))
        with pytest.raises(NotImplementedError):
            UNetSpatioTemporalConditionModel()  # class default heads (5, 10, 10, 20): 128-wide heads in stage 3


def test_router_state_dict_and_config():
    from oracle.adapter import ControlNetRouter as O
    ours, ref = A.ControlNetRouter(**cases.ROUTER_KW), O(**cases.ROUTER_KW)
    assert set(ours.state_dict()) == set(ref.state_dict())
    assert ours.router_type == "simple_weights" and ours.num_routers == 12 and ours.num_experts == 7
    with pytest.raises(ValueError):
        A.ControlNetRouter(router_type="sparsemax")


def test_timestep_vector_forms():
    from ctrl_adapter_b200.layers import timestep_vector
    dev = torch.device("cpu")
    for t in (981, 981.0, torch.tensor(981.0), torch.tensor([981.0]), torch.tensor([[981.0], [981.0], [981.0]])):
        v = timestep_vector(t, 3, dev)
        assert v.shape == (3,) and v.dtype == torch.float32 and float(v[0]) == 981.0
    with pytest.raises(TypeError):
        timestep_vector("981", 3, dev)


def test_adapter_rejects_unsupported_configs():
    with pytest.raises(NotImplementedError):
        A.ControlNetAdapter("sdxl", num_repeats=2, add_adapter_location_A=True)
    with pytest.raises(ValueError):
        A.AdapterSpatioTemporal(320, 640)


def test_adapter_save_load_roundtrip(tmp_path):
    kw = dict(cases.ADAPTER_SDXL_KW, add_adapter_location_B=False, add_adapter_location_C=False,
              num_adapters_per_location=1)
    m = A.ControlNetAdapter(**kw)
    m.save_pretrained(str(tmp_path / "adapter"))
    m2 = A.ControlNetAdapter.from_pretrained(str(tmp_path), subfolder="adapter")
    assert m2.config == m.config
    for (k1, v1), (k2, v2) in zip(m.state_dict().items(), m2.state_dict().items()):
        assert k1 == k2 and torch.equal(v1, v2)


def test_pretrained_folder_roundtrip(tmp_path):
    """save_pretrained -> from_pretrained (config.json + safetensors / .bin) for the small boundary classes, and config
    reconstruction of every class from its own saved configuration and from the published checkpoints' config.json."""
    import json
    import os
    from ctrl_adapter_b200.controlnet import ControlNetModel
    from ctrl_adapter_b200.unet_i2vgen import I2VGenXLUNet
    from ctrl_adapter_b200.unet_sdxl import UNet2DConditionModel
    from ctrl_adapter_b200.unet_svd import UNetSpatioTemporalConditionModel
    r = A.ControlNetRouter(**cases.ROUTER_KW)
    for safe in (True, False):
        d = str(tmp_path / f"router{int(safe)}")
        r.save_pretrained(d, safe_serialization=safe)
        assert json.load(open(os.path.join(d, "config.json")))["_class_name"] == "ControlNetRouter"
        r2 = A.ControlNetRouter.from_pretrained(str(tmp_path), subfolder=f"router{int(safe)}", low_cpu_mem_usage=False,
                                                device_map=None)
        assert r2.router_type == r.router_type and r2.num_experts == r.num_experts
        for (k1, v1), (k2, v2) in zip(r.state_dict().items(), r2.state_dict().items()):
            assert k1 == k2 and torch.equal(v1, v2)
    with pytest.raises(FileNotFoundError):
        A.ControlNetRouter.from_pretrained(str(tmp_path / "missing"))
    # published config.json contents (abridged to the keys that matter + a few the classes must tolerate)
    published = {
        ControlNetModel: dict(_class_name="ControlNetModel", _diffusers_version="0.16.0.dev0", act_fn="silu",
                              attention_head_dim=8, block_out_channels=[320, 640, 1280, 1280], class_embed_type=None,
                              conditioning_embedding_out_channels=[16, 32, 96, 256],
                              controlnet_conditioning_channel_order="rgb", cross_attention_dim=768,
                              down_block_types=["CrossAttnDownBlock2D"] * 3 + ["DownBlock2D"], downsample_padding=1,
                              flip_sin_to_cos=True, freq_shift=0, in_channels=4, layers_per_block=2,
                              mid_block_scale_factor=1, norm_eps=1e-05, norm_num_groups=32, num_class_embeds=None,
                              only_cross_attention=False, projection_class_embeddings_input_dim=None,
                              resnet_time_scale_shift="default", upcast_attention=False, use_linear_projection=False),
        UNet2DConditionModel: dict(_class_name="UNet2DConditionModel", act_fn="silu", addition_embed_type="text_time",
                                   addition_time_embed_dim=256, attention_head_dim=[5, 10, 20],
                                   block_out_channels=[320, 640, 1280], cross_attention_dim=2048, in_channels=4,
                                   out_channels=4, projection_class_embeddings_input_dim=2816, sample_size=128,
                                   transformer_layers_per_block=[1, 2, 10], use_linear_projection=True,
                                   down_block_types=["DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D"]),
        I2VGenXLUNet: dict(_class_name="I2VGenXLUNet", attention_head_dim=64, block_out_channels=[320, 640, 1280, 1280],
                           cross_attention_dim=1024, in_channels=4, out_channels=4, layers_per_block=2,
                           norm_num_groups=32, num_attention_heads=None, sample_size=32,
                           down_block_types=["CrossAttnDownBlock3D"] * 3 + ["DownBlock3D"],
                           up_block_types=["UpBlock3D"] + ["CrossAttnUpBlock3D"] * 3),
        UNetSpatioTemporalConditionModel: dict(_class_name="UNetSpatioTemporalConditionModel", addition_time_embed_dim=256,
                                               block_out_channels=[320, 640, 1280, 1280], cross_attention_dim=1024,
                                               in_channels=8, layers_per_block=2, num_attention_heads=[5, 10, 20, 20],
                                               num_frames=14, out_channels=4, projection_class_embeddings_input_dim=768,
                                               sample_size=96, transformer_layers_per_block=1,
                                               down_block_types=["CrossAttnDownBlockSpatioTemporal"] * 3 +
                                               ["DownBlockSpatioTemporal"],
                                               up_block_types=["UpBlockSpatioTemporal"] +
                                               ["CrossAttnUpBlockSpatioTemporal"] * 3),
    }
    with torch.device("meta"):
        for cls, cfg in published.items():
            m = cls.from_config(cfg)
            m2 = cls.from_config(json.loads(json.dumps({"_class_name": cls.__name__, **dict(m.config)}, default=list)))
            assert set(m.state_dict()) == set(m2.state_dict())


def test_reference_import_paths_resolve():
    """SURVEY.md section 8b: the module paths AND NAMES inference.py imports (:351-367) exist and resolve to the H100-backed
    classes (or, for the out-of-scope helpers, to stubs that fail loudly when used)."""
    import argparse
    from controlnet.controlnet import ControlNetModel  # noqa: F401
    from controlnet.multicontrolnet import MultiControlNetModel  # noqa: F401
    from i2vgen_xl.models.unets.unet_i2vgen_xl import I2VGenXLUNet  # noqa: F401
    from i2vgen_xl.pipelines.i2vgen_xl_controlnet_adapter_pipeline import I2VGenXLControlNetAdapterPipeline  # noqa: F401
    from model.ctrl_adapter import ControlNetAdapter  # noqa: F401
    from model.ctrl_helper import ControlNetHelper
    from model.ctrl_router import ControlNetRouter  # noqa: F401
    from sdxl.pipelines.sdxl_controlnet_adapter_pipeline import SDXLControlNetAdapterPipeline  # noqa: F401
    from svd.models.unets.unet_spatio_temporal_condition import UNetSpatioTemporalConditionModel  # noqa: F401
    from svd.pipelines.svd_controlnet_adapter_pipeline import SVDControlNetAdapterPipeline  # noqa: F401
    from utils.utils import bool_flag, center_crop_and_resize, save_as_gif, save_concatenated_gif  # noqa: F401
    assert ControlNetAdapter is A.ControlNetAdapter
    assert bool_flag("True") is True and bool_flag("off") is False
    with pytest.raises(argparse.ArgumentTypeError):
        bool_flag("maybe")
    helper = ControlNetHelper()  # no hub access: constructed without a text encoder
    with pytest.raises(NotImplementedError):
        helper.add_depth_estimator()
    with pytest.raises(NotImplementedError):
        helper.encode_controlnet_prompt("a cat", "cpu", 1, True)
    with pytest.raises(NotImplementedError):
        save_as_gif([], "x.gif")


def test_controlnet_keep_is_the_reference_formula():
    """loop_base.controlnet_keep / control_scale against the literal comprehension of the reference
    (sdxl_controlnet_adapter_pipeline.py:1207-1211, :1296-1302) for the shipped settings (start 0, end 0.5 / 0.6 / 1)."""
    from ctrl_adapter_b200.loop_base import DenoiseLoopBase, controlnet_keep
    for n, s, e in [(50, 0.0, 0.5), (50, 0.0, 0.6), (25, 0.0, 0.4), (4, 0.0, 0.5), (50, 0.2, 1.0), (7, 0.1, 0.9)]:
        ref = [[1.0 - float(i / n < s_ or (i + 1) / n > e_) for s_, e_ in zip([s], [e])] for i in range(n)]
        assert controlnet_keep(n, [s], [e]) == ref
    loop = DenoiseLoopBase()
    loop.num_inference_steps = 50
    loop._init_control(0.75, 0.0, 0.6, 1)
    assert [loop.control_scale(i) for i in (0, 29, 30, 49)] == [0.75, 0.75, 0.0, 0.0]
    loop._init_control([1.0, 0.5], 0.0, [1.0, 0.5], 2)  # Multi-ControlNet: one keep per net, scale stays a tuple
    assert loop.control_scale(10) == (1.0, 0.5) and loop.control_scale(40) == (1.0, 0.0)


def test_static_context_cache_hits_only_the_registered_tensor():
    """Attention.cache_static / cache_static_context: the stored K/V is used for the registered tensor OBJECT while it is
    unmodified, and recomputed for a clone, after an in-place update, and after the weights change."""
    from tests import ops_emulator as emu
    from ctrl_adapter_b200.layers import Attention, cache_static_context
    torch.manual_seed(0)
    att = Attention(128, 96, 2, 64).to(torch.bfloat16)
    x = torch.randn(2, 16, 128).to(torch.bfloat16)
    ctx = torch.randn(2, 5, 96).to(torch.bfloat16)
    calls = []
    with emu.patched_ops():
        orig = att.project_kv
        att.project_kv = lambda c: (calls.append(1), orig(c))[1]
        assert cache_static_context(att, ctx) == 1 and len(calls) == 1
        y0 = att(x, ctx=ctx)
        assert len(calls) == 1                       # hit
        y1 = att(x, ctx=ctx.clone())
        assert len(calls) == 2                       # another tensor object: recomputed
        assert torch.equal(y0, y1)
        ctx.mul_(2.0)
        y2 = att(x, ctx=ctx)
        assert len(calls) == 3 and not torch.equal(y0, y2)   # in-place update seen through _version
        cache_static_context(att, ctx)
        with torch.no_grad():
            att.to_q.weight.add_(1.0)                # first parameter changes -> _key() changes -> stale entry ignored
        att(x, ctx=ctx)
        assert len(calls) == 5


def test_pipeline_classes_mirror_the_reference_signatures():
    """The three pipeline classes take the reference's constructor and __call__ parameters, in the reference's order
    (names extracted from /root/reference with ast by the snippet in tests/golden/README, committed as
    tests/golden/reference_pipeline_signatures.json); ours may only APPEND keyword extensions."""
    import inspect
    import json
    import os
    from ctrl_adapter_b200 import pipelines as P
    ref = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "reference_pipeline_signatures.json")))
    for cls_name, fns in ref.items():
        cls = getattr(P, cls_name)
        for fn, names in fns.items():
            ours = [n for n in inspect.signature(getattr(cls, fn)).parameters if n not in ("self", "kwargs")]
            assert ours[: len(names)] == names, (cls_name, fn, [a for a in zip(ours, names) if a[0] != a[1]][:3])
            if fn == "__init__":
                assert len(ours) == len(names)


def test_pipeline_needs_pre_encoded_inputs_without_encoders():
    """Without encoder components the pipeline asks for the pre-encoded tensors instead of silently doing something
    else; component registry / to() / from_pretrained error path."""
    from ctrl_adapter_b200 import pipelines as P
    pipe = P.SDXLControlNetAdapterPipeline(vae=None, text_encoder=None, text_encoder_2=None, tokenizer=None,
                                           tokenizer_2=None, unet=torch.nn.Linear(1, 1), scheduler=None, adapter=None,
                                           helper=None, controlnet=torch.nn.Linear(1, 1))
    assert set(pipe.components) >= {"unet", "controlnet", "adapter", "helper", "vae"}
    assert pipe.to(torch.float32) is pipe and pipe.device.type == "cpu"
    with pytest.raises(ValueError, match="prompt_embeds"):
        pipe(prompt="a cat", control_images=torch.zeros(1, 3, 512, 512))
    with pytest.raises(FileNotFoundError):
        P.SDXLControlNetAdapterPipeline.from_pretrained("/nonexistent/snapshot", controlnet=None, adapter=None, helper=None)


def test_helper_prepare_images_batched_and_prompt_encoding():
    """ControlNetHelper.prepare_images (ctrl_helper.py:268-296) for PIL / ndarray / tensor frames and batch sizes > 1, and
    encode_controlnet_prompt (:301-457) on a duck-typed tokenizer / text encoder."""
    import numpy as np
    from PIL import Image
    from ctrl_adapter_b200.helper import ControlNetHelper
    h = ControlNetHelper()
    rng = np.random.default_rng(0)
    frames = [Image.fromarray(rng.integers(0, 255, (40, 60, 3), dtype=np.uint8)) for _ in range(3)]
    out = h.prepare_images(frames, 32, 16, batch_size=2, num_images_per_prompt=1, device="cpu", dtype=torch.float32,
                           do_classifier_free_guidance=True)
    assert out.shape == (2, 6, 3, 16, 32) and 0.0 <= float(out.min()) and float(out.max()) <= 1.0
    assert torch.equal(out[0], out[1]) and torch.equal(out[0, :3], out[0, 3:])   # CFG copy, batch repeat
    ref0 = np.array(frames[0].convert("RGB").resize((32, 16), resample=Image.LANCZOS)).astype(np.float32) / 255.0
    assert np.allclose(out[0, 0].permute(1, 2, 0).numpy(), ref0)
    t = h.prepare_images([torch.rand(3, 16, 32), rng.random((16, 32, 3)).astype(np.float32)], 32, 16, 1, 1, "cpu",
                         torch.float32)
    assert t.shape == (1, 2, 3, 16, 32)

    class Tok:
        model_max_length = 5

        def __call__(self, text, padding, max_length, truncation, return_tensors):
            text = [text] if isinstance(text, str) else text
            ids = torch.tensor([[len(s) % 7] * max_length for s in text])
            return type("E", (), {"input_ids": ids, "attention_mask": torch.ones_like(ids)})()

    class Enc(torch.nn.Module):
        dtype = torch.float32

        def forward(self, ids, attention_mask=None, output_hidden_states=False):
            e = ids.float().unsqueeze(-1).repeat(1, 1, 4)
            return (e, e.mean(1))

    h2 = ControlNetHelper(text_encoder=Enc(), tokenizer=Tok())
    pe, ne, pp, npp = h2.encode_controlnet_prompt(["ab", "abc"], "cpu", 2, True)
    assert pe.shape == (4, 5, 4) and ne.shape == (4, 5, 4) and pp.shape == (4, 4) and npp.shape == (4, 4)
    assert float(ne.abs().max()) == 0.0 and float(pe[0, 0, 0]) == 2.0 and float(pe[2, 0, 0]) == 3.0
    assert h2._get_add_time_ids((1024, 1024), (0, 0), (1024, 1024), torch.float32).shape == (1, 6)
