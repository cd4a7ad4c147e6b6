"""DenseCorrespondenceNetwork -- same public surface as the reference's
dense_correspondence/network/dense_correspondence_network.py (class at :21), with the backbone
running in libddn_b200.so.

Kept verbatim in behaviour: ``forward`` (:239-263), ``forward_single_image_tensor`` (:265-299),
``process_network_output`` (:303-319), ``get_fcn`` (:360-383), ``from_config`` (:386-438),
``from_model_folder`` (:441-485), ``find_best_match`` (:488-525), ``descriptor_image_stats`` (:136-152) and the
properties training.py / evaluation.py read.  Left out (not on the hot path, need the dataset stack / PIL / utils
module): ``load_training_dataset``, ``get_unet`` -- they raise NotImplementedError.
"""
import logging
import os
import warnings

import numpy as np
import torch
import torch.nn as nn
import yaml

from . import resnet_dilated


class DenseCorrespondenceNetwork(nn.Module):

    def __init__(self, fcn, descriptor_dimension, image_width=640, image_height=480, normalize=False):
        super(DenseCorrespondenceNetwork, self).__init__()
        self._fcn = fcn
        self._descriptor_dimension = descriptor_dimension
        self._image_width = image_width
        self._image_height = image_height
        # identity by default: the dataset loader normalises the images (net.py:52, spartan_dataset_masked.py:297-304)
        self._image_mean = np.zeros(3)
        self._image_std_dev = np.ones(3)
        self.config = dict()
        self._descriptor_image_stats = None
        self._normalize = normalize
        self._constructed_from_model_folder = False

    @property
    def fcn(self):
        return self._fcn

    @property
    def config(self):
        return self._config

    @config.setter
    def config(self, value):
        self._config = value

    @property
    def descriptor_dimension(self):
        return self._descriptor_dimension

    @property
    def image_shape(self):
        return [self._image_height, self._image_width]

    @property
    def image_mean(self):
        return self._image_mean

    @image_mean.setter
    def image_mean(self, value):
        self._image_mean = value
        self.config['image_mean'] = value

    @property
    def image_std_dev(self):
        return self._image_std_dev

    @image_std_dev.setter
    def image_std_dev(self, value):
        self._image_std_dev = value
        self.config['image_std_dev'] = value

    @property
    def path_to_network_params_folder(self):
        if 'path_to_network_params_folder' not in self.config:
            raise ValueError("DenseCorrespondenceNetwork: Config doesn't have a `path_to_network_params_folder`"
                             "entry")
        return self.config['path_to_network_params_folder']

    @property
    def constructed_from_model_folder(self):
        return self._constructed_from_model_folder

    @constructed_from_model_folder.setter
    def constructed_from_model_folder(self, value):
        self._constructed_from_model_folder = value

    @property
    def descriptor_image_stats(self):
        """net.py:136-152: descriptor_statistics.yaml of the network's parameter folder (written by
        evaluation.save_descriptor_statistics), loaded on first use.  A relative folder is taken relative to the home
        directory, as utils.convert_to_absolute_path does."""
        if self._descriptor_image_stats is None:
            path = self.path_to_network_params_folder
            if not os.path.isdir(path):
                path = os.path.join(os.path.expanduser("~"), path)
            with open(os.path.join(path, "descriptor_statistics.yaml")) as f:
                self._descriptor_image_stats = yaml.safe_load(f)
        return self._descriptor_image_stats

    def load_training_dataset(self):
        raise NotImplementedError("the SpartanDataset stack is out of scope (SURVEY.md 2a #5)")

    def forward(self, img_tensor):
        """[N,3,H,W] fp32 CUDA (already normalised) -> [N,D,H,W] fp32, contiguous NCHW (net.py:239-263)."""
        res = self.fcn(img_tensor)
        if self._normalize:
            # net.py:256-259 -- as written upstream this only broadcasts for N == 1; kept, not fixed
            tag = resnet_dilated.lowres_of(res)
            norm = torch.norm(res, 2, 1)
            res = res / norm
            if tag is not None and res.shape[0] == 1:   # per pixel at N == 1: a fused loss normalises the blend the same way
                resnet_dilated.attach_lowres(res, tag[0], tag[1], tag[2], unit=True)
        return res

    def forward_pair(self, img_a, img_b, per_pixel_normalize=False):
        """(image_a_pred, image_b_pred) = (self.forward(img_a), self.forward(img_b)) -- the two forward calls of a reference
        training step (dense_correspondence/training/training.py:329-333) -- executed as ONE launch sequence over the
        concatenated batch with two BatchNorm groups: each image batch is normalised by its own batch statistics and the
        running statistics are updated A-then-B, exactly as the two calls would, but every kernel runs once on twice the
        pixels (half the launches, better SM fill) and there is a single backward.  Opt-in: the reference API is two calls.

        ``per_pixel_normalize=True`` (only on a network built with ``normalize``): every pixel of every image is divided by
        its own L2 norm, as each of the reference's batch-1 calls does (net.py:256-259), at any batch size.  Like
        ``forward_pair`` itself this is the project's batched generalisation; the upsample kernel writes the unit descriptors
        and the fused loss normalises its blended descriptors the same way.  A zero descriptor gives NaN, as in the
        reference.  The default keeps the reference expression, which only broadcasts per pixel for a batch of one."""
        if img_a.shape != img_b.shape:
            raise ValueError("forward_pair needs two image batches of the same shape")
        if per_pixel_normalize and not self._normalize:
            raise ValueError("per_pixel_normalize=True needs a network built with normalize=True")
        B = img_a.shape[0]
        if per_pixel_normalize:
            res = self.fcn(torch.cat([img_a, img_b], 0), bn_groups=2, per_pixel_normalize=True)
        else:
            res = self.fcn(torch.cat([img_a, img_b], 0), bn_groups=2)
        res_a, res_b = res[:B], res[B:]
        tag = resnet_dilated.lowres_of(res)
        if tag is not None:
            resnet_dilated.attach_lowres(res_a, tag[0][:B], tag[1], tag[2], unit=tag[4])
            resnet_dilated.attach_lowres(res_b, tag[0][B:], tag[1], tag[2], unit=tag[4])
        if self._normalize and not per_pixel_normalize:
            res_a = res_a / torch.norm(res_a, 2, 1)
            res_b = res_b / torch.norm(res_b, 2, 1)
            if tag is not None and B == 1:      # per pixel at B == 1: a fused loss normalises the blend the same way
                resnet_dilated.attach_lowres(res_a, tag[0][:B], tag[1], tag[2], unit=True)
                resnet_dilated.attach_lowres(res_b, tag[0][B:], tag[1], tag[2], unit=True)
        return res_a, res_b

    def forward_single_image_tensor(self, img_tensor):
        """[3,H,W] -> [H,W,D] (net.py:265-299)."""
        assert len(img_tensor.shape) == 3
        img_tensor = img_tensor.unsqueeze(0)
        img_tensor = img_tensor.detach().to(device=torch.device("cuda"), dtype=torch.float32).contiguous()
        res = self.forward(img_tensor)
        res = res.squeeze(0)
        res = res.permute(1, 2, 0)
        return res

    def forward_on_img_tensor(self, img):
        warnings.warn("use forward method instead", DeprecationWarning)
        return self.forward_single_image_tensor(img).data.cpu().numpy().squeeze()

    def process_network_output(self, image_pred, N):
        """[N,D,H,W] -> strided view [N, W*H, D] (net.py:303-319)."""
        W = self._image_width
        H = self._image_height
        tag = resnet_dilated.lowres_of(image_pred)
        image_pred = image_pred.view(N, self.descriptor_dimension, W * H)
        image_pred = image_pred.permute(0, 2, 1)
        if tag is not None:       # a view of the same storage (shares the version counter): the tag stays valid
            resnet_dilated.attach_lowres(image_pred, tag[0], tag[1], tag[2], unit=tag[4])
        return image_pred

    def clip_pixel_to_image_size_and_round(self, uv):
        u = min(int(round(uv[0])), self._image_width - 1)
        v = min(int(round(uv[1])), self._image_height - 1)
        return [u, v]

    @staticmethod
    def get_unet(config):
        raise NotImplementedError("the Unet backbone is not part of this hot path (net.py:346-357)")

    @staticmethod
    def get_fcn(config):
        """net.py:360-383.  Resnet34_8s and Resnet50_8s exist in this build; anything else raises (no fallback)."""
        if config["backbone"]["model_class"] == "Resnet":
            resnet_model = config["backbone"]["resnet_name"]
            if resnet_model not in ("Resnet34_8s", "Resnet50_8s"):
                raise ValueError("backbone %s is not implemented in this path (only Resnet34_8s and Resnet50_8s)" % resnet_model)
            fcn = getattr(resnet_dilated, resnet_model)(num_classes=config['descriptor_dimension'])
        elif config["backbone"]["model_class"] == "Unet":
            fcn = DenseCorrespondenceNetwork.get_unet(config)
        else:
            raise ValueError("Can't build backbone network.  I don't know this backbone model class!")
        return fcn

    @staticmethod
    def from_config(config, load_stored_params=True, model_param_file=None):
        """net.py:386-438."""
        if "backbone" not in config:
            config["backbone"] = dict()
            config["backbone"]["model_class"] = "Resnet"
            config["backbone"]["resnet_name"] = "Resnet34_8s"
        fcn = DenseCorrespondenceNetwork.get_fcn(config)
        normalize = config['normalize'] if 'normalize' in config else False
        dcn = DenseCorrespondenceNetwork(fcn, config['descriptor_dimension'],
                                         image_width=config['image_width'],
                                         image_height=config['image_height'],
                                         normalize=normalize)
        if load_stored_params:
            assert model_param_file is not None
            config['model_param_file'] = model_param_file
            state = torch.load(model_param_file, map_location="cpu")
            try:
                dcn.load_state_dict(state)
            except Exception:
                logging.info("loading params with the new style failed, falling back to dcn.fcn.load_state_dict")
                dcn.fcn.load_state_dict(state)
        dcn.cuda()
        dcn.train()
        dcn.config = config
        return dcn

    @staticmethod
    def from_model_folder(model_folder, load_stored_params=True, model_param_file=None, iteration=None):
        """net.py:441-485 (utils.get_model_param_file_from_directory restated: newest / requested NNNNNN.pth)."""
        from_model_folder = False
        model_folder = os.path.abspath(os.path.expanduser(model_folder))
        if model_param_file is None:
            cands = sorted(f for f in os.listdir(model_folder) if f.endswith(".pth"))
            if not cands:
                raise ValueError("no .pth file in %s" % model_folder)
            if iteration is None:
                model_param_file = os.path.join(model_folder, cands[-1])
            else:
                want = "%06d.pth" % iteration
                if want not in cands:
                    raise ValueError("%s not found in %s" % (want, model_folder))
                model_param_file = os.path.join(model_folder, want)
            from_model_folder = True
        model_param_file = os.path.abspath(model_param_file)
        with open(os.path.join(model_folder, "training.yaml")) as f:
            training_config = yaml.safe_load(f)
        config = training_config["dense_correspondence_network"]
        config["path_to_network_params_folder"] = model_folder
        config["model_param_filename_tail"] = os.path.split(model_param_file)[1]
        dcn = DenseCorrespondenceNetwork.from_config(config, load_stored_params=load_stored_params,
                                                     model_param_file=model_param_file)
        dcn.constructed_from_model_folder = from_model_folder
        dcn.model_folder = model_folder
        return dcn

    @staticmethod
    def find_best_match(pixel_a, res_a, res_b, debug=False):
        """net.py:488-525: numpy argmin of the descriptor distance (host-side, as in the reference)."""
        descriptor_at_pixel = res_a[pixel_a[1], pixel_a[0]]
        norm_diffs = np.sqrt(np.sum(np.square(res_b - descriptor_at_pixel), axis=2))
        best_match_flattened_idx = np.argmin(norm_diffs)
        best_match_xy = np.unravel_index(best_match_flattened_idx, norm_diffs.shape)
        best_match_diff = norm_diffs[best_match_xy]
        best_match_uv = (best_match_xy[1], best_match_xy[0])
        return best_match_uv, best_match_diff, norm_diffs

    @staticmethod
    def find_best_matches_cuda(pixels_a, res_a, res_b, return_norm_diffs=False, mask_b=None):
        """Device-side, batched ``find_best_match`` (net.py:488-525): ``pixels_a`` [Q,2] (u,v) integer pixels in image A,
        ``res_a`` / ``res_b`` [H,W,D] float32 CUDA descriptor images (what ``forward_single_image_tensor`` returns, any
        strides).  -> (best_uv [Q,2] int64 CUDA, best_diff [Q] float32 CUDA[, norm_diffs [Q,H,W]]) without leaving the
        GPU; evaluation.py:993,1047 does this 100x per pair on the host after a D2H copy.  ``mask_b`` ([H,W], 1 on the
        object): the result tuple is extended by (best_uv_masked [Q,2], best_diff_masked [Q]) = the argmin of
        ``norm_diffs + (1 - mask_b) * 1e6`` (evaluation.py:1052-1059), from the same pass."""
        from . import _native as N
        N.require_cuda_f32(res_a, "res_a", contiguous=False); N.require_cuda_f32(res_b, "res_b", contiguous=False)
        H, W, D = res_b.shape
        if res_b.stride(0) != W * res_b.stride(1):
            res_b = res_b.contiguous()
        px = torch.as_tensor(pixels_a, dtype=torch.long, device=res_a.device).reshape(-1, 2)
        q = res_a[px[:, 1], px[:, 0]].contiguous()                      # [Q, D] query descriptors
        Q = q.shape[0]
        uv = torch.empty(Q, 2, dtype=torch.int64, device=res_b.device)
        diff = torch.empty(Q, dtype=torch.float32, device=res_b.device)
        nd = torch.empty(Q, H, W, dtype=torch.float32, device=res_b.device) if return_norm_diffs else None
        scratch = torch.empty(2 * Q, dtype=torch.int64, device=res_b.device)
        mk = uvm = diffm = None
        if mask_b is not None:
            mk = torch.as_tensor(mask_b).to(device=res_b.device, dtype=torch.float32).reshape(H * W).contiguous()
            uvm = torch.empty(Q, 2, dtype=torch.int64, device=res_b.device)
            diffm = torch.empty(Q, dtype=torch.float32, device=res_b.device)
        N.check(N.lib.ddn_find_best_match(N.ptr(res_b), res_b.stride(1), res_b.stride(2), H, W, D, N.ptr(q), Q, N.ptr(uv),
                                          N.ptr(diff), N.ptr(nd), N.ptr(mk), N.ptr(uvm), N.ptr(diffm), N.ptr(scratch),
                                          N.stream_ptr()))
        out = (uv, diff, nd) if return_norm_diffs else (uv, diff)
        return out + (uvm, diffm) if mask_b is not None else out

    @staticmethod
    def find_best_match_for_descriptor(descriptor, res):
        norm_diffs = np.sqrt(np.sum(np.square(res - descriptor), axis=2))
        best_match_flattened_idx = np.argmin(norm_diffs)
        best_match_xy = np.unravel_index(best_match_flattened_idx, norm_diffs.shape)
        best_match_diff = norm_diffs[best_match_xy]
        best_match_uv = (best_match_xy[1], best_match_xy[0])
        return best_match_uv, best_match_diff, norm_diffs
