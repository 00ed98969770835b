"""Host-side mirrors of the reference's scoring helpers, on the C ABI's device primitives:

  sort_images_by_prediction   NN_UTILS.sortImagesByPrediction (utils/nn_utils.lua:90-118; sample.lua:84-85)
  find_closest_neighbours     findClosestNeighboursOf (sample.lua:141-159)
  approx_parzen               adversarial.approxParzen (adversarial_c2f.lua:305-325)
"""
import ctypes as C

import numpy as np

from .lib import _check, f32


def d_score(ctx, images, chunk, training=True, seed=0):
    images = f32(images)
    preds = np.empty(images.shape[0], np.float32)
    _check(ctx.lib.fg_D_score(ctx.h, images.ctypes.data_as(C.c_void_p), images.shape[0], chunk, int(training), seed,
                              preds.ctypes.data_as(C.c_void_p)), "fg_D_score")
    return preds


def sort_images_by_prediction(ctx, images, ascending, nb_max_out, chunk, training=True, seed=0):
    """-> (images, predictions): the nb_max_out images D rates most fake (ascending) / most real first."""
    preds = d_score(ctx, images, chunk, training, seed)
    order = np.argsort(preds if ascending else -preds, kind="stable")[:nb_max_out]
    return np.asarray(images)[order], preds[order]


def nearest(ctx, queries, cands):
    queries, cands = f32(queries), f32(cands)
    Q, N = queries.shape[0], cands.shape[0]
    D = int(np.prod(queries.shape[1:]))
    idx, dist = np.empty(Q, np.int32), np.empty(Q, np.float32)
    _check(ctx.lib.fg_nearest(ctx.h, queries.ctypes.data_as(C.c_void_p), Q, cands.ctypes.data_as(C.c_void_p), N, D,
                              idx.ctypes.data_as(C.c_void_p), dist.ctypes.data_as(C.c_void_p)), "fg_nearest")
    return idx, dist


def find_closest_neighbours(dataset, images):
    """-> list of (image, closest training image (32x32 float), distance) like sample.lua:141-159."""
    images = f32(images)
    Q = images.shape[0]
    idx, dist = np.empty(Q, np.int32), np.empty(Q, np.float32)
    _check(dataset.lib.fg_dataset_nearest(dataset.h, images.ctypes.data_as(C.c_void_p), Q, idx.ctypes.data_as(C.c_void_p),
                                          dist.ctypes.data_as(C.c_void_p)), "fg_dataset_nearest")
    neigh = dataset.gather(idx)
    return [(images[i], neigh[i], float(dist[i])) for i in range(Q)], idx


def approx_parzen(net, fine, coarse, nneighbors, rng):
    """distances[n] = min_k || G({noise_k, coarse_n}) + coarse_n - fine_n || for every (fine, coarse) pair given."""
    fine, coarse = f32(fine), f32(coarse)
    out = np.empty(fine.shape[0], np.float32)
    d = np.empty(1, np.float32)
    for i in range(fine.shape[0]):
        noise = rng.uniform(-1, 1, (nneighbors, 1, net.S, net.S)).astype(np.float32)
        _check(net.lib.fg_c2f_parzen_dist(net.h, noise.ctypes.data_as(C.c_void_p), coarse[i].ctypes.data_as(C.c_void_p),
                                          fine[i].ctypes.data_as(C.c_void_p), nneighbors, d.ctypes.data_as(C.c_void_p)),
               "fg_c2f_parzen_dist")
        out[i] = d[0]
    return out
