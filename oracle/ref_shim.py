"""TEST INFRASTRUCTURE ONLY -- loader for the *reference's own* dense path.

Imports the reference's Python files in place from ``/root/reference`` (read-only, present in
the build container only -- it does NOT exist on the GPU box) so that ``oracle/restated.py`` can
be pinned against the real thing and golden vectors can be generated
(``tests/golden/make_golden.py``).  Nothing in the product path may import this module.

The reference cannot be imported as-is here (SURVEY.md section 8c): ``llavamod/__init__.py``
eagerly imports every model family and needs deepspeed / transformers==4.37.  Four harness
shims make the *dense* path (vendored Qwen1.5 + CLIP tower + projector + multimodal splice)
importable without touching the reference tree:

1. pre-register empty ``llavamod`` and ``llavamod.model`` (+ sub-packages) in ``sys.modules``
   with ``__path__`` set, so their ``__init__.py`` never execute;
2. stub ``timm.models.vision_transformer.Block`` (imported by the unused simple/pool projector
   blocks, ``multimodal_projector/simple_block.py:5``);
3. transformers>=5 auto-generates ``__init__`` for config subclasses -> restore
   ``LlavaQwen1_5Config.__init__ = Qwen2Config.__init__``;
4. ``config.pad_token_id = None`` (read at ``qwen1_5/modeling_qwen2.py:942``).
"""
import importlib
import os
import sys
import types

REF_ROOT = os.environ.get("LLAVAMOD_REFERENCE", "/root/reference")


def available() -> bool:
    return os.path.isdir(os.path.join(REF_ROOT, "llavamod", "model"))


def _pkg(name, path):
    if name in sys.modules:
        return sys.modules[name]
    m = types.ModuleType(name)
    m.__path__ = [path]
    m.__package__ = name
    sys.modules[name] = m
    return m


_loaded = {}


def load():
    """Returns a namespace with the reference classes of the dense path.

    The reference uses absolute ``llavamod.*`` imports, so it has to live under that name in ``sys.modules`` -- the same
    name as this project's package.  The two therefore never share a process: tests reach the reference through
    ``run_child`` (a subprocess running ``oracle/ref_child.py``); only ``tests/golden/make_golden.py`` and that child
    call ``load()`` directly."""
    if "llavamod" in sys.modules and not getattr(sys.modules["llavamod"], "__path__", [""])[0].startswith(REF_ROOT):
        raise RuntimeError("this project's llavamod package is already imported in this process; use ref_shim.run_child()")
    if _loaded:
        return types.SimpleNamespace(**_loaded)
    if not available():
        raise RuntimeError("reference tree not present at %s" % REF_ROOT)
    base = os.path.join(REF_ROOT, "llavamod")
    _pkg("llavamod", base)
    _pkg("llavamod.model", os.path.join(base, "model"))
    _pkg("llavamod.model.language_model", os.path.join(base, "model", "language_model"))
    _pkg("llavamod.model.language_model.qwen1_5", os.path.join(base, "model", "language_model", "qwen1_5"))
    _pkg("llavamod.model.multimodal_encoder", os.path.join(base, "model", "multimodal_encoder"))
    _pkg("llavamod.model.multimodal_projector", os.path.join(base, "model", "multimodal_projector"))
    # shim 2: timm stub
    if "timm" not in sys.modules:
        try:
            import timm  # noqa: F401
        except Exception:
            import torch.nn as nn
            import importlib.machinery as _mach

            def _stub(name, pkg=False):
                mod = types.ModuleType(name)
                mod.__spec__ = _mach.ModuleSpec(name, None, is_package=pkg)   # transformers probes find_spec("timm")
                if pkg:
                    mod.__path__ = []
                return mod

            t = _stub("timm", True)
            tm = _stub("timm.models", True)
            tv = _stub("timm.models.vision_transformer")
            tl = _stub("timm.models.layers")
            tml = _stub("timm.layers")

            class Block(nn.Module):  # never instantiated on the dense path
                pass

            tv.Block = Block
            for mod in (tl, tml):
                mod.LayerNorm2d = nn.LayerNorm
                mod.LayerNorm = nn.LayerNorm
                mod.trunc_normal_ = nn.init.trunc_normal_
                mod.DropPath = nn.Identity
                mod.Mlp = nn.Identity
            tr = _stub("timm.models.regnet")
            tr.RegStage = Block
            sys.modules.update({"timm": t, "timm.models": tm, "timm.models.vision_transformer": tv,
                                "timm.models.layers": tl, "timm.layers": tml, "timm.models.regnet": tr})
    # the encoder / projector builders import sibling files explicitly
    enc_builder = importlib.import_module("llavamod.model.multimodal_encoder.builder")
    clip_enc = importlib.import_module("llavamod.model.multimodal_encoder.clip_encoder")
    proj_builder = importlib.import_module("llavamod.model.multimodal_projector.builder")
    arch = importlib.import_module("llavamod.model.llava_arch")
    mq = importlib.import_module("llavamod.model.language_model.qwen1_5.modeling_qwen2")
    lq = importlib.import_module("llavamod.model.language_model.llava_qwen1_5")
    consts = importlib.import_module("llavamod.constants")
    # shim 3
    lq.LlavaQwen1_5Config.__init__ = mq.Qwen2Config.__init__
    _loaded.update(dict(enc_builder=enc_builder, clip_encoder=clip_enc, proj_builder=proj_builder,
                        llava_arch=arch, modeling_qwen2=mq, llava_qwen1_5=lq, constants=consts))
    return types.SimpleNamespace(**_loaded)


def build_tiny_dense(tmpdir, hidden=128, inter=256, layers=2, heads=4, kv_heads=4, vocab=512,
                     clip_hidden=64, clip_inter=128, clip_layers=3, clip_heads=4, image=32, patch=8,
                     rope_theta=1e6, seed=0, attn="sdpa"):
    """Instantiates the reference's LlavaQwen1_5ForCausalLM (dense teacher class,
    llava_qwen1_5.py:56-167) with a tiny random CLIP tower saved under a directory whose name
    contains "openai" (multimodal_encoder/builder.py:25 dispatches on that substring)."""
    import torch
    from transformers import CLIPVisionConfig, CLIPVisionModel, CLIPImageProcessor
    ref = load()
    torch.manual_seed(seed)
    clip_dir = os.path.join(tmpdir, "openai-tiny-clip")
    if not os.path.isdir(clip_dir):
        ccfg = CLIPVisionConfig(hidden_size=clip_hidden, intermediate_size=clip_inter,
                                num_hidden_layers=clip_layers, num_attention_heads=clip_heads,
                                image_size=image, patch_size=patch, hidden_act="quick_gelu",
                                layer_norm_eps=1e-5, projection_dim=clip_hidden)
        cm = CLIPVisionModel(ccfg)
        cm.save_pretrained(clip_dir)
        CLIPImageProcessor(size={"shortest_edge": image}, crop_size={"height": image, "width": image}
                           ).save_pretrained(clip_dir)
    cfg = ref.llava_qwen1_5.LlavaQwen1_5Config(
        vocab_size=vocab, hidden_size=hidden, intermediate_size=inter, num_hidden_layers=layers,
        num_attention_heads=heads, num_key_value_heads=kv_heads, max_position_embeddings=512,
        rope_theta=rope_theta, rms_norm_eps=1e-6, tie_word_embeddings=False, use_sliding_window=False,
        attention_dropout=0.0)
    cfg.pad_token_id = None  # shim 4
    cfg.use_cache = False  # training sets this (align_train.py); transformers-5 DynamicCache lacks the legacy API
    cfg._attn_implementation = attn
    model = ref.llava_qwen1_5.LlavaQwen1_5ForCausalLM(cfg)
    margs = types.SimpleNamespace(image_tower=clip_dir, video_tower=None, mm_vision_select_layer=-2,
                                  mm_vision_select_feature="patch", pretrain_mm_mlp_adapter=None,
                                  image_projector_type="mlp2x_gelu", video_projector_type="linear",
                                  video_global_proj=False, video_temproal_proj=False,
                                  video_spatial_proj=False)
    model.get_model().initialize_vision_modules(margs)
    model.eval()
    return model


def run_child(request: dict, timeout=600):
    """Runs oracle/ref_child.py in a clean subprocess (reference namespace isolated from this project's package).
    ``request`` = dict(kw=<build_tiny_dense kwargs>, input_ids, labels, attention_mask, images, padding_side).
    Returns dict(state_dict, logits, labels, loss)."""
    import subprocess
    import tempfile
    import torch
    d = tempfile.mkdtemp()
    req, resp = os.path.join(d, "req.pt"), os.path.join(d, "resp.pt")
    torch.save(request, req)
    env = dict(os.environ)
    env["PYTHONPATH"] = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, os.path.join(os.path.dirname(os.path.abspath(__file__)), "ref_child.py"), req, resp],
                       capture_output=True, text=True, timeout=timeout, env=env)
    if r.returncode != 0:
        raise RuntimeError("reference child failed:\n" + r.stdout[-2000:] + r.stderr[-4000:])
    return torch.load(resp, weights_only=False)
