"""Command-line programs with the reference's interfaces, on the native trainers and renderers:

    python -m gms_b200.cli.train   -s <scene> -m <output> --gs_type gs_mesh|gs_flat|gs     train.py
    python -m gms_b200.cli.render  -m <output> --gs_type gs_mesh|gs_flat|gs|gs_points      scripts/render.py
    python -m gms_b200.cli.metrics -m <output> [<output> ...] --gs_type ...               metrics.py (LPIPS with --lpips)

and the reference's scripts/ for trained models (gs_multi_mesh and gs_flame render through cli.render as well):

    python -m gms_b200.cli.render_time_animated        -m <output>                       scripts/render_time_animated.py
    python -m gms_b200.cli.render_points_time_animated -m <output>                       scripts/render_points_time_animated.py
    python -m gms_b200.cli.render_from_object          -m <output> --object_path <obj>   scripts/render_from_object.py
    python -m gms_b200.cli.render_flame                -m <output> [--animated]          scripts/render_flame.py
    python -m gms_b200.cli.render_multi_mesh           -m <output>                       scripts/render_multi_mesh.py
    python -m gms_b200.cli.render_from_mesh_to_mesh    -m <output> --target_mesh <obj>   scripts/render_from_mesh_to_mesh.py
    python -m gms_b200.cli.save_pseudomesh             --model_path <output>             scripts/save_pseudomesh.py
    python -m gms_b200.cli.create_dummy_mesh           --pseudomesh_path <triangles.pt>  scripts/create_dummy_mesh.py
    python -m gms_b200.cli.edit_pseudomesh             --triangle_soup_path ... --save_dir ...
                                                                          scripts/edit_pseudomesh_based_on_estimated_mesh.py

and the server side of the SIBR remote viewer (renderer/gaussian_renderer/network_gui.py) for a trained model:

    python -m gms_b200.cli.view                        -m <output> [--ip 127.0.0.1] [--port 6009]

Each module has main(argv), which the tests call in-process."""
