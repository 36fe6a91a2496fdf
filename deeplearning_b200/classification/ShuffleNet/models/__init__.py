from .shufflenetv1 import model_dict, get_model
# from .shufflenetv2 import model_dict, get_model
