from .shufflenetv1 import model_dict, get_model
