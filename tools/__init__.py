import os


def output_path(name: str) -> str:
    """Path of a check / probe report: under $LAH_CHECK_OUT (default: check_out/ in the working directory)."""
    out_dir = os.environ.get("LAH_CHECK_OUT", "check_out")
    os.makedirs(out_dir, exist_ok=True)
    return os.path.join(out_dir, name)
