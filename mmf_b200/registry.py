"""Minimal mirror of `mmf.common.registry.registry` for the registration calls this path uses
(mmf/common/registry.py:296-322, 369-375, 423-451, 542-608, and register_scheduler).  With a real MMF install the same decorators are taken
from `mmf.common.registry`; this shim exists because the reference package cannot be imported in this environment
(omegaconf / pytorch_lightning missing, SURVEY.md 8c)."""


class Registry:
    mapping = {"model_name_mapping": {}, "encoder_name_mapping": {}, "transformer_backend_name_mapping": {},
               "processor_name_mapping": {}, "scheduler_name_mapping": {}, "state": {}}

    @classmethod
    def _register(cls, table, name):
        def wrap(obj):
            cls.mapping[table][name] = obj
            return obj
        return wrap

    @classmethod
    def register_model(cls, name):
        return cls._register("model_name_mapping", name)

    @classmethod
    def register_encoder(cls, name):
        return cls._register("encoder_name_mapping", name)

    @classmethod
    def register_transformer_backend(cls, name):
        return cls._register("transformer_backend_name_mapping", name)

    @classmethod
    def register_processor(cls, name):
        return cls._register("processor_name_mapping", name)

    @classmethod
    def register_scheduler(cls, name):
        return cls._register("scheduler_name_mapping", name)

    @classmethod
    def get_model_class(cls, name):
        return cls.mapping["model_name_mapping"].get(name, None)

    @classmethod
    def get_encoder_class(cls, name):
        return cls.mapping["encoder_name_mapping"].get(name, None)

    @classmethod
    def get_transformer_backend_class(cls, name):
        return cls.mapping["transformer_backend_name_mapping"].get(name, None)

    @classmethod
    def get_processor_class(cls, name):
        return cls.mapping["processor_name_mapping"].get(name, None)

    @classmethod
    def get_scheduler_class(cls, name):
        return cls.mapping["scheduler_name_mapping"].get(name, None)

    @classmethod
    def register(cls, name, obj):
        cls.mapping["state"][name] = obj

    @classmethod
    def get(cls, name, default=None):
        return cls.mapping["state"].get(name, default)


registry = Registry()
