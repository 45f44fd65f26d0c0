"""`python -m animate3d_b200.mesh2gaussian --input_obj M.obj --output_dir D --output_name N`: the engine's replacement for
tools/mesh_animation/mesh2gaussian.py, with its flags and file names (D/N.ply, D/N.json)."""
from __future__ import annotations

import argparse

from .mesh import write_mesh_gaussians


def main(argv=None) -> None:
    p = argparse.ArgumentParser(description="Convert OBJ to Gaussian point cloud and extract connected vertices info.")
    p.add_argument("--input_obj", required=True, help="Path to input OBJ file")
    p.add_argument("--output_dir", required=True, help="Directory to save output files")
    p.add_argument("--output_name", required=True, help="Base name for output files (without extension)")
    a = p.parse_args(argv)
    ply, js = write_mesh_gaussians(a.input_obj, a.output_dir, a.output_name)
    print(f"Gaussian point cloud saved to {ply}")
    print(f"Connected vertices information saved to {js}")


if __name__ == "__main__":
    main()
