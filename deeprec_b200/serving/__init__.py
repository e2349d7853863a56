from .export import (export_delta, export_delta_module, export_delta_program, export_saved_model, export_saved_model_module,  # noqa: F401
                     export_saved_model_program, export_zoo_model, export_engine_program, export_engine_delta,
                     load_zoo_model, compress_sample_aware, taobao_user_columns)
from .processor import Processor, ProcessorGroup, decode_response, encode_request  # noqa: F401
from .session_group import SessionGroup  # noqa: F401
