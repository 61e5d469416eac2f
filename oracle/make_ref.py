"""Recipe that stages the REFERENCE's own, unmodified Python modules for this path under oracle/_ref/ so that the timed CPU baseline
(`bench.py --impl reference`, `cpu_baseline`) runs the reference's stock code instead of the oracle port.

    python oracle/make_ref.py            # needs a checkout of the reference (R3DP_REFERENCE); machines without it use the staged files

Nothing is edited: the files are byte-for-byte copies, found as the import closure of the reference classes on the path
(ImportanceRenderer, RaySampler, OSGDecoder, SuperresolutionHybrid8XDC, SuperresolutionHybrid8XDC_Warp).  oracle/_ref/ is git-ignored
(reference sources never enter this repository's history).
Test infrastructure: only tests/, __graft_entry__ and bench.py's CPU-baseline legs may touch oracle/."""
import hashlib
import json
import os
import shutil
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get('R3DP_REFERENCE', '/root/reference')
DST = os.path.join(HERE, '_ref')


def closure(with_torso_head: bool = True):
    """Files of the reference tree imported by the classes on the path."""
    sys.path.insert(0, REF)
    sys.modules.setdefault('imageio', types.ModuleType('imageio'))          # utils/commons/image_utils.py:7 imports it; never called on this path
    before = set(sys.modules)
    from utils.commons.hparams import hparams
    hparams.update(dict(enable_rescale_plane_regulation=False, triplane_feature_type='triplane', triplane_depth=1))
    import modules.eg3ds.volumetric_rendering.renderer       # noqa: F401
    import modules.eg3ds.volumetric_rendering.ray_sampler    # noqa: F401
    import modules.eg3ds.models.triplane                     # noqa: F401
    import modules.eg3ds.models.superresolution              # noqa: F401
    import modules.eg3ds.camera_utils.pose_sampler           # noqa: F401
    if with_torso_head:
        try:
            import modules.real3d.super_resolution.sr_with_ref   # noqa: F401
        except Exception as e:                                   # noqa: BLE001
            print('torso head not staged:', type(e).__name__, e)
    files = set()
    for name in set(sys.modules) - before:
        f = getattr(sys.modules[name], '__file__', None)
        if f and os.path.abspath(f).startswith(os.path.abspath(REF) + os.sep):
            files.add(os.path.abspath(f))
    return sorted(files)


def main():
    if not os.path.isdir(REF):
        print(f'{REF} not present: keeping whatever oracle/_ref already holds')
        return 0
    files = closure()
    if os.path.isdir(DST):
        shutil.rmtree(DST)
    manifest = {}
    for f in files:
        rel = os.path.relpath(f, REF)
        out = os.path.join(DST, rel)
        os.makedirs(os.path.dirname(out), exist_ok=True)
        shutil.copyfile(f, out)
        manifest[rel] = hashlib.sha256(open(f, 'rb').read()).hexdigest()[:16]
    json.dump({'source': REF, 'files': manifest}, open(os.path.join(DST, 'MANIFEST.json'), 'w'), indent=1, sort_keys=True)
    print(f'staged {len(files)} reference files under {DST}')
    return 0


if __name__ == '__main__':
    sys.exit(main())
