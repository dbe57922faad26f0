"""renderih_b200 -- H100-native (sm_90a) hot path of adwardlee/RenderIH: HandNET_GCN forward/backward + ManoLayer.

Public API mirrors the reference modules it replaces:
    load_model(cfg) / HandNET_GCN      <-  models/model.py:18-60
    ManoLayer, rodrigues_batch          <-  models/manolayer.py:32-48,100-322
    load_graph_model(cfg)               <-  common/myhand/lijun_model_graph.py:37-70 (the trainers' default model)
    load_new_model(cfg)                 <-  common/myhand/lijun_model_newgraph.py:34-71 (graph model + MANO tail)
    preprocess_u8(frames, flip)         <-  core/loader.py:151-152,178-181 (host image ops of the loader, on the GPU)
    augment_u8 / get_affine_mat / prepare_labels  <-  core/loader.py:96-211, utils/manoutils.py:183-261 (training-time augmentation:
                                            cv2.warpAffine, brightness noise, flip, normalisation in one kernel; label transforms)
    calc_loss_GCN / mano_loss_GCN       <-  core/Loss.py:201-277, core/Loss_mano.py:245-335 (fused mesh-term kernels, loss.py)
    Jr, batch_metrics, EvalMetrics      <-  apps/eval_interhand.py:28-170,300-552, utils/eval_metrics.py:36-50 (metrics.py)
    TrainStep, lr_at_epoch              <-  core/lijun_trainer.py:131-159,262-313, utils/lr_sc.py:159-175 (train.py)
    mano_two_hands_renderer, rasterize, hand_mask_iou  <-  utils/vis_utils.py:153-289, utils/compute_maskiou.py:59-64,250-263 (render.py:
                                            pytorch3d rasterise + hard Phong / ambient shading, per-sample hand mask IoU)
    NewLoss, SDF                        <-  pose_data_optimize/code_sdf/sdf_template.py:19-157, lib/sdf/sdf/sdf.py (sdf.py: two-hand
                                            anti-penetration loss of the pose optimiser and its dense SDF grid; the function
                                            `sdf` is renderih_b200.sdf.sdf, since the submodule owns that name)
    manopth.ManoLayer                   <-  pose_data_optimize/manopth/manopth/manolayer.py (the pose optimiser's quaternion hand model,
                                            quat/quat without PCA; a submodule only, since the top-level name ManoLayer is taken)
    geo_loss.AnchorLayer, HandPriorLoss <-  pose_data_optimize/manopth/manopth/anchorlayer.py, hocontact/postprocess/geo_loss.py (the pose
                                            optimiser's anchor layer and its quat-norm, edge, contact and ergonomics terms for both hands)
    Pos2dDiscriminator, NatureLoss      <-  pose_data_optimize/Ver2Code/Discriminator/discrim.py:66-105, hocontact/postprocess/
                                            geo_optimizer_both_batch.py:110-132 (nature.py: the pose optimiser's discriminator and its
                                            nature loss on both hands, with the pose gradient)
    GeOptimizer                         <-  pose_data_optimize/hocontact/postprocess/geo_optimizer_both_batch.py:22-930 (ge_optimizer.py:
                                            the two-hand pose optimiser, set_opt_val / optimize, one CUDA graph per iteration with
                                            device-side Adam and ReduceLROnPlateau)
    hand_collision_count, filter_collision_data  <-  pose_data_optimize/collision/CollisionFilter.py:9-127, CollisionCheck.py
                                            (collision.py: per-frame count of intersecting face pairs between the two hand meshes)
    ValidJudger, get_valid_rate         <-  pose_data_optimize/Ver2Code/ValidJudge/ValidJudger.py, GetValidRate.py (valid_judge.py:
                                            the joint-limit validity rate of both hands)
    HandPoseConverter, HandPoseArguer, PoseArguer, convert_annotations, argue_data, reconvert_optimized, birth_data
                                        <-  pose_data_optimize/scripts/HandPoseConverter.py, HandPoseArguer.py, Ver2Code/NatureJudge/
                                            PoseArgue.py, data_birth.py, data/template_{0,1,3}_*.py (pose_data.py: euler / MANO
                                            quaternion / axis-angle conversions and pose augmentation, one launch per batch)
    HeatmapGenerator, cut_img, InterHandLoader, select_data, cut_inter_img, InterHand_dataset, render_data
                                        <-  dataset/heatmap.py, dataset/dataset_utils.py, utils/dataset_gen/interhand.py,
                                            rendering_code/step7_gen_annotations.py (dataset_gen.py: batched crops, annotations,
                                            ori_handdict labels, heatmaps, masks and dense maps)
"""
from . import _build


def build(force=False):
    """Compile the CUDA library for sm_90a (in-tree)."""
    return _build.build(force=force)


def __getattr__(name):
    if name in ('load_model', 'HandNET_GCN', 'load_encoder', 'load_decoder'):
        from . import model
        return getattr(model, name)
    if name in ('ManoLayer', 'rodrigues_batch'):
        from . import manolayer
        return getattr(manolayer, name)
    if name in ('load_graph_model', 'load_new_model'):
        from . import myhand
        return getattr(myhand, name)
    if name in ('preprocess_u8', 'augment_u8', 'get_affine_mat', 'augment_labels', 'prepare_labels'):
        from . import input as _input
        return getattr(_input, name)
    if name in ('GraphLoss', 'ManoLoss', 'calc_loss_GCN', 'mano_loss_GCN'):
        from . import loss
        return getattr(loss, name)
    if name in ('Jr', 'batch_metrics', 'EvalMetrics'):
        from . import metrics
        return getattr(metrics, name)
    if name in ('TrainStep', 'FlatParams', 'lr_at_epoch'):
        from . import train
        return getattr(train, name)
    if name in ('mano_two_hands_renderer', 'rasterize', 'hand_mask_iou'):
        from . import render
        return getattr(render, name)
    if name in ('NewLoss', 'SDF'):
        from . import sdf as _sdf
        return getattr(_sdf, name)
    if name in ('Pos2dDiscriminator', 'NatureLoss'):
        from . import nature
        return getattr(nature, name)
    if name == 'GeOptimizer':
        from . import ge_optimizer
        return ge_optimizer.GeOptimizer
    if name in ('hand_collision_count', 'filter_collision_data'):
        from . import collision
        return getattr(collision, name)
    if name in ('ValidJudger', 'get_valid_rate'):
        from . import valid_judge
        return getattr(valid_judge, name)
    if name in ('HandPoseConverter', 'HandPoseArguer', 'PoseArguer', 'convert_annotations', 'argue_data', 'reconvert_optimized', 'birth_data'):
        from . import pose_data
        return getattr(pose_data, name)
    if name in ('HeatmapGenerator', 'cut_img', 'InterHandLoader', 'select_data', 'cut_inter_img', 'InterHand_dataset', 'render_data'):
        from . import dataset_gen
        return getattr(dataset_gen, name)
    if name in ('load_cfg', 'get_cfg_defaults'):
        from . import config
        return getattr(config, name)
    raise AttributeError(name)
