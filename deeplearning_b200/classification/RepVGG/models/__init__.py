from .repvgg import get_RepVGG_func_by_name, func_dict, repvgg_model_convert  # noqa: F401
