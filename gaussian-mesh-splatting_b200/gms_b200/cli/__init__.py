"""Command-line programs with the reference's interfaces, on the native trainers and renderers:

    python -m gms_b200.cli.train   -s <scene> -m <output> --gs_type gs_mesh|gs_flat|gs     train.py
    python -m gms_b200.cli.render  -m <output> --gs_type gs_mesh|gs_flat|gs|gs_points      scripts/render.py
    python -m gms_b200.cli.metrics -m <output> [<output> ...] --gs_type ...               metrics.py (LPIPS with --lpips)

Each module has main(argv), which the tests call in-process."""
