"""mmf_b200 - H100-native (sm_90a) fusion block for MMF-style multimodal transformers.

Importing the package loads libmmfb200.so (building it in-tree with nvcc if missing) and fails loudly if that is
impossible; there is no CPU fallback for any compute path.  See DESIGN.md / INTEGRATION.md.

    from mmf_b200 import B200BertEncoder, B200ViLBertEncoder, B200VisualBERT, replace_with_b200
"""
__version__ = "0.1.0"

_LAZY = {
    "B200BertEncoder": ("modules", "B200BertEncoder"),
    "B200ViLBertEncoder": ("modules", "B200ViLBertEncoder"),
    "B200VisioLinguisticEmbeddings": ("embeddings", "B200VisioLinguisticEmbeddings"),
    "B200VisualBERT": ("visual_bert", "B200VisualBERT"),
    "B200VisualBERTBase": ("visual_bert", "B200VisualBERTBase"),
    "B200VisualBERTForPretraining": ("visual_bert", "B200VisualBERTForPretraining"),
    "B200BertPreTrainingHeads": ("heads", "B200BertPreTrainingHeads"),
    "B200AdamW": ("optim", "B200AdamW"),
    "B200MMBTBase": ("mmbt", "B200MMBTBase"),
    "B200MMBTModel": ("mmbt", "B200MMBTModel"),
    "B200ViLBERTBase": ("vilbert", "B200ViLBERTBase"),
    "B200TransformerBackend": ("mmft_backend", "B200TransformerBackend"),
    "B200UNITERModelBase": ("uniter", "B200UNITERModelBase"),
    "B200LXMERTEncoder": ("lxmert", "B200LXMERTEncoder"),
    "B200TransformerEncoder": ("encoders", "B200TransformerEncoder"),
    "B200FinetuneFasterRcnnFpnFc7": ("encoders", "B200FinetuneFasterRcnnFpnFc7"),
    "B200IdentityEncoder": ("encoders", "B200IdentityEncoder"),
    "build_encoder": ("encoders", "build_encoder"),
    "B200DataParallel": ("ddp", "B200DataParallel"),
    "replace_with_b200": ("patch", "replace_with_b200"),
    "undo_replace_with_b200": ("patch", "undo_replace_with_b200"),
    "attach_encoder": ("patch", "attach_encoder"),
    "SampleList": ("sample", "SampleList"),
    "VisualBERT": ("models", "VisualBERT"),
    "ViLBERT": ("models", "ViLBERT"),
    "MMBT": ("models", "MMBT"),
    "MMFTransformer": ("mmft", "MMFTransformer"),
    "UNITER": ("uniter_model", "UNITER"),
    "VinVL": ("vinvl_model", "VinVL"),
    "ViLT": ("vilt_model", "ViLT"),
    "M4C": ("m4c_model", "M4C"),
    "M4CCaptioner": ("m4c_model", "M4CCaptioner"),
    "build_model": ("models", "build_model"),
    "load_model_config": ("models", "load_model_config"),
    "GraphedStep": ("graphs", "GraphedStep"),
    "GraphedForward": ("graphs", "GraphedForward"),
}


def __getattr__(name):
    if name in _LAZY:
        import importlib
        mod, attr = _LAZY[name]
        return getattr(importlib.import_module("." + mod, __name__), attr)
    raise AttributeError("module %r has no attribute %r" % (__name__, name))
