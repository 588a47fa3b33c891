#!/bin/bash
# A/B the render kernel across prebuilt library variants (diagnostic).
for lib in build_variants/lib_*.so; do
  echo "$lib"; MP_ENGINE_LIB=$PWD/$lib python tools/render_bound.py | cut -c1-400
done
