"""A synthetic stage-2 folder for device position maps: the folder of dataset_fixture.write_synthetic_dataset without inp_map/, with
the full SMPL mesh model (posedirs [6890,3,207], weights, f) in SMPL_NEUTRAL.pkl and the synthetic UV template at
project/assets/template_mesh_smpl_uv.obj.  Test helper, not product."""
import os
import pickle
from os.path import join

from dataset_fixture import write_synthetic_dataset
from gaussianavatar_b200 import synthetic as syn


def write_posmap_dataset(root, seed=0, **kw):
    """Returns ModelParams with train_stage=2 and inp_posmap_from_pose=True."""
    mp = write_synthetic_dataset(root, seed=seed, stage2=False, **kw)
    template = syn.make_uv_template(seed)
    with open(join(mp.smpl_model_path, "SMPL_NEUTRAL.pkl"), "wb") as f:
        pickle.dump(syn.smpl_mesh_model(syn.make_body(seed), template), f)
    syn.write_uv_template_obj(join(mp.project_path, "assets", "template_mesh_smpl_uv.obj"), template)
    mp.train_stage = 2
    mp.inp_posmap_from_pose = True
    return mp
