from dynaboa_b200.render import Renderer, convert_crop_cam_to_orig_img  # noqa: F401
