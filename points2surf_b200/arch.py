"""Parameter inventory of PointsToSurfModel (names / shapes / registration order), derived from the
module structure of source/points_to_surf_model.py:12-36,72-99,134-167,237-294."""


def head_output_dim(outputs):
    """The supported `--outputs` lists of a checkpoint, shared by training and evaluation so that every checkpoint the
    training writes can be evaluated: -> 1 for the regression head (imp_surf), 2 for magnitude + sign; else ValueError."""
    outs = list(outputs)
    if 'imp_surf' in outs:
        # the regression ablation (experiments/*_p2s_regression.sh); the reference's save_evaluation indexes the
        # patch_pts_ids and p_index outputs (points_to_surf_eval.py:287-288), so it needs them too
        if 'imp_surf_magnitude' in outs or 'imp_surf_sign' in outs or outs.count('imp_surf') > 1:
            raise ValueError('Unsupported outputs %s: imp_surf together with imp_surf_magnitude / imp_surf_sign' % outs)
        if 'patch_pts_ids' not in outs or 'p_index' not in outs:
            raise ValueError('Unsupported outputs %s: imp_surf needs patch_pts_ids and p_index' % outs)
        return 1
    if 'imp_surf_magnitude' not in outs or 'imp_surf_sign' not in outs:
        raise ValueError('Unsupported outputs %s: need imp_surf_magnitude + imp_surf_sign, or imp_surf' % outs)
    return 2


def layer_specs(use_point_stn, shared_transformation, net=1024, output_dim=2, single_transformer=False):
    """-> list of (dotted name, kind in {'conv','fc','bn'}, cout, cin) in state_dict order.
    single_transformer: the shared encoder (source/points_to_surf_model.py:253-263): feat_local_global (its QSTN iff
    use_point_stn), fc1_local_global (net -> net), bn1_local_global, then the common head; shared_transformation plays
    no part."""

    def stn(prefix, dim, quat):
        out = 4 if quat else dim * dim
        return [(prefix + 'conv1', 'conv', 64, dim), (prefix + 'conv2', 'conv', 128, 64),
                (prefix + 'conv3', 'conv', net, 128),
                (prefix + 'fc1', 'fc', net // 2, net), (prefix + 'fc2', 'fc', net // 4, net // 2),
                (prefix + 'fc3', 'fc', out, net // 4),
                (prefix + 'bn1', 'bn', 64, 0), (prefix + 'bn2', 'bn', 128, 0), (prefix + 'bn3', 'bn', net, 0),
                (prefix + 'bn4', 'bn', net // 2, 0), (prefix + 'bn5', 'bn', net // 4, 0)]

    def feat(prefix, point_stn):
        s = []
        if point_stn:
            s += stn(prefix + 'stn1.', 3, True)
        s += stn(prefix + 'stn2.', 64, False)
        s += [(prefix + 'conv0a', 'conv', 64, 3), (prefix + 'conv0b', 'conv', 64, 64),
              (prefix + 'bn0a', 'bn', 64, 0), (prefix + 'bn0b', 'bn', 64, 0),
              (prefix + 'conv1', 'conv', 64, 64), (prefix + 'conv2', 'conv', 128, 64),
              (prefix + 'conv3', 'conv', net, 128),
              (prefix + 'bn1', 'bn', 64, 0), (prefix + 'bn2', 'bn', 128, 0), (prefix + 'bn3', 'bn', net, 0)]
        return s

    specs = []
    if single_transformer:
        specs += feat('feat_local_global.', bool(use_point_stn))
        specs += [('fc1_local_global', 'fc', net, net), ('bn1_local_global', 'bn', net, 0)]
    else:
        if use_point_stn and shared_transformation:
            specs += stn('point_stn.', 3, True)
        specs += feat('feat_local.', False)
        specs += feat('feat_global.', bool(use_point_stn and not shared_transformation))
        specs += [('fc1_local', 'fc', net // 2, net), ('fc1_global', 'fc', net // 2, net),
                  ('bn1_local', 'bn', net // 2, 0), ('bn1_global', 'bn', net // 2, 0)]
    specs += [('fc2', 'fc', net // 4, net), ('fc3', 'fc', net // 8, net // 4), ('fc4', 'fc', output_dim, net // 8),
              ('bn2', 'bn', net // 4, 0), ('bn3', 'bn', net // 8, 0)]
    return specs
