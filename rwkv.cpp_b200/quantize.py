"""Quantizes an rwkv.cpp model file from FP32 or FP16 (CLI of the reference's python/quantize.py:8-32 over this library's
rwkv_quantize_model_file, which is byte-identical to the reference's for all seven formats and needs no GPU; the one exception: a
Q4_K / Q5_K tensor whose rows are not whole 256-weight super-blocks is written as Q5_0 / Q5_1, where the reference writes blocks that
straddle rows).

    python rwkv.cpp_b200/quantize.py model-FP16.bin model-Q5_1.bin Q5_1
"""
import argparse
import importlib.util
import os
import sys

FORMAT_NAMES = ("Q4_0", "Q4_1", "Q4_K", "Q5_0", "Q5_1", "Q5_K", "Q8_0")      # the reference binding's list, in its order


def _load_package():
    if "rwkv_cpp_b200" in sys.modules:
        return sys.modules["rwkv_cpp_b200"]
    here = os.path.dirname(os.path.abspath(__file__))
    spec = importlib.util.spec_from_file_location("rwkv_cpp_b200", os.path.join(here, "__init__.py"), submodule_search_locations=[here])
    mod = importlib.util.module_from_spec(spec)
    sys.modules["rwkv_cpp_b200"] = mod
    spec.loader.exec_module(mod)
    return mod


def main(argv=None) -> None:
    ap = argparse.ArgumentParser(description="Quantize rwkv.cpp model file from FP32 or FP16")
    ap.add_argument("src_path", help="Path to FP32/FP16 checkpoint file")
    ap.add_argument("dest_path", help="Path to resulting checkpoint file, will be overwritten")
    ap.add_argument("format_name", help="Format name, one of " + ", ".join(FORMAT_NAMES), choices=FORMAT_NAMES, default="Q5_1", nargs="?")
    args = ap.parse_args(argv)
    library = _load_package().load_rwkv_shared_library()
    library.rwkv_quantize_model_file(args.src_path, args.dest_path, args.format_name)
    print("Done")


if __name__ == "__main__":
    main()
