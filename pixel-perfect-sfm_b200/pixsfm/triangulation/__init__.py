from .main import (DEFAULT_MAPPER_OPTIONS, main, mapper_options_from, pack_matches, read_inputs,  # noqa: F401
                   triangulate_points, unique_pairs)
