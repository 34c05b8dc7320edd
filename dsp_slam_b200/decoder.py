"""Ingest a DeepSDF decoder the way DSP-SLAM hands it over and upload it to the GPU library.

The reference passes the `nn.Module` returned by reconstruct.utils.get_decoder
(deep_sdf/workspace.py:202-223) into Optimizer / MeshExtractor.  This module pulls the Linear
(and LayerNorm) layers out of such a module (or out of a state_dict / npz fixture), folds weight-norm once
(W = g * v / ||v||_row, torch.nn.utils.weight_norm(dim=0) as applied at
deep_sdf/deep_sdf_decoder.py:49-56), records the decoder's structural options (latent_in, xyz_in_all, use_tanh)
and creates the device-resident decoder handle.
"""
import ctypes as C
import json
import numpy as np

from . import _lib


class DecoderWeights:
    """Folded fp32 weights of one decoder: W[k] (out,in), b[k] (out,), latent size L, and what
    deep_sdf_decoder.py concatenates at each layer's input -- cat_kind[k]: 0 nothing, 1 the decoder input
    (`latent_in`, :87-88), 2 xyz (`xyz_in_all`, :89-90) -- plus the optional LayerNorm (gamma, beta) after layer k
    (:58-63,96-102) and `use_tanh` (:93-94).  Accepted: 3 to 9 linear layers, each at most 512 wide, a latent size of
    at most 64.  The plain shape (one latent_in layer, nothing else) with every layer at most 256 wide runs on the
    tensor-core engine; every other decoder -- a variant, or a layer wider than 256 such as DeepSDF's own 8 x 512
    network -- on the fp32 SIMT engine."""

    def __init__(self, W, b, latent_in, latent_size, xyz_in_all=False, use_tanh=False, ln=None):
        self.W = [np.ascontiguousarray(w, dtype=np.float32) for w in W]
        self.b = [np.ascontiguousarray(x, dtype=np.float32) for x in b]
        self.latent_in = tuple(int(i) for i in (latent_in or ()))
        self.latent_size = int(latent_size)
        self.xyz_in_all = bool(xyz_in_all)
        self.use_tanh = bool(use_tanh)
        n = len(self.W)
        self.ln = list(ln) if ln is not None else [None] * n
        self.cat_kind = [1 if k in self.latent_in else (2 if (k != 0 and self.xyz_in_all) else 0) for k in range(n)]
        self.latent_in_layer = self.latent_in[0] if len(self.latent_in) == 1 else -1
        in0 = self.latent_size + 3
        if self.W[0].shape[1] != in0:
            raise ValueError("first layer must take latent_size+3 inputs")
        for k in range(1, n):
            want = self.W[k - 1].shape[0] + (in0 if self.cat_kind[k] == 1 else (3 if self.cat_kind[k] == 2 else 0))
            if self.W[k].shape[1] != want:
                raise ValueError(f"layer {k}: in_dim {self.W[k].shape[1]} does not match the decoder structure ({want})")

    @property
    def is_plain(self):
        return (not self.xyz_in_all and not self.use_tanh and all(x is None for x in self.ln)
                and len(self.latent_in) <= 1 and all(k <= len(self.W) - 2 for k in self.latent_in))

    # -- constructors ------------------------------------------------------------------------
    @staticmethod
    def _fold(sd, k):
        if f"lin{k}.weight_v" in sd:
            v = np.asarray(sd[f"lin{k}.weight_v"], dtype=np.float32)
            g = np.asarray(sd[f"lin{k}.weight_g"], dtype=np.float32).reshape(-1, 1)
            norm = np.sqrt(np.sum(v * v, axis=1, keepdims=True, dtype=np.float32))
            return (g * (v / norm)).astype(np.float32)
        if f"lin{k}.parametrizations.weight.original1" in sd:      # new-style parametrization
            v = np.asarray(sd[f"lin{k}.parametrizations.weight.original1"], dtype=np.float32)
            g = np.asarray(sd[f"lin{k}.parametrizations.weight.original0"], dtype=np.float32).reshape(-1, 1)
            norm = np.sqrt(np.sum(v * v, axis=1, keepdims=True, dtype=np.float32))
            return (g * (v / norm)).astype(np.float32)
        return np.asarray(sd[f"lin{k}.weight"], dtype=np.float32)

    @classmethod
    def from_state_dict(cls, sd, latent_size, latent_in=(), xyz_in_all=None, use_tanh=False, latent_dropout=False):
        """latent_dropout is a training-time option (F.dropout with training=False is the identity, :80-83)."""
        sd = {k: (v.detach().cpu().numpy() if hasattr(v, "detach") else np.asarray(v)) for k, v in sd.items()}
        n_lin = 0
        while any(k.startswith(f"lin{n_lin}.") for k in sd):
            n_lin += 1
        W = [cls._fold(sd, k) for k in range(n_lin)]
        b = [np.asarray(sd[f"lin{k}.bias"], dtype=np.float32) for k in range(n_lin)]
        ln = [(np.asarray(sd[f"bn{k}.weight"], dtype=np.float32), np.asarray(sd[f"bn{k}.bias"], dtype=np.float32))
              if f"bn{k}.weight" in sd else None for k in range(n_lin)]
        return cls(W, b, latent_in, latent_size, xyz_in_all=bool(xyz_in_all), use_tanh=bool(use_tanh), ln=ln)

    @classmethod
    def from_module(cls, module):
        """`module` = deep_sdf.deep_sdf_decoder.Decoder (eval).  Attributes used: latent_in, xyz_in_all, use_tanh,
        state_dict() (lin{k}.weight[_g/_v] / bias, bn{k}.weight / bias)."""
        sd = module.state_dict()
        L = None
        for key in ("lin0.weight_v", "lin0.weight", "lin0.parametrizations.weight.original1"):
            if key in sd:
                L = int(sd[key].shape[1]) - 3
        if L is None:
            raise ValueError("module has no lin0 layer")
        return cls.from_state_dict(sd, L, latent_in=tuple(getattr(module, "latent_in", ()) or ()),
                                   xyz_in_all=getattr(module, "xyz_in_all", None),
                                   use_tanh=getattr(module, "use_tanh", False))

    @classmethod
    def from_npz(cls, path):
        d = np.load(path)
        spec = json.loads(bytes(d["spec_json"]).decode())
        sd = {k: d[k] for k in d.files if k != "spec_json"}
        return cls.from_state_dict(sd, spec["latent_size"], latent_in=spec.get("latent_in", ()),
                                   xyz_in_all=spec.get("xyz_in_all"), use_tanh=spec.get("use_tanh"))

    @classmethod
    def coerce(cls, obj):
        if isinstance(obj, cls):
            return obj
        if isinstance(obj, str):
            return cls.from_npz(obj)
        if hasattr(obj, "state_dict"):
            return cls.from_module(obj)
        raise TypeError(f"cannot build decoder weights from {type(obj)}")


class DeviceDecoder:
    """Owns a DspgnDecoder handle (weights resident in HBM in every layout the kernels use)."""

    def __init__(self, weights, device=0):
        lib = _lib.load()
        self.weights = weights
        self.device = device
        spec = _lib.DecoderSpec()
        spec.latent_size = weights.latent_size
        spec.num_linear = len(weights.W)
        if spec.num_linear > _lib.MAX_LINEAR:
            raise ValueError("too many layers")
        for k, w in enumerate(weights.W):
            spec.out_dim[k], spec.in_dim[k] = w.shape
        spec.latent_in_layer = weights.latent_in_layer
        for k in range(spec.num_linear):
            spec.cat_kind[k] = weights.cat_kind[k]
            spec.layer_norm[k] = 1 if weights.ln[k] is not None else 0
        spec.use_tanh = int(weights.use_tanh)
        FP = C.POINTER(C.c_float)
        Wp = (FP * len(weights.W))(*[w.ctypes.data_as(FP) for w in weights.W])
        bp = (FP * len(weights.b))(*[x.ctypes.data_as(FP) for x in weights.b])
        n = len(weights.W)
        self._ln_keep = [(np.ascontiguousarray(g, np.float32), np.ascontiguousarray(be, np.float32)) if (g is not None) else (None, None)
                         for g, be in [(x if x is not None else (None, None)) for x in weights.ln]]
        gp = (FP * n)(*[(g.ctypes.data_as(FP) if g is not None else None) for g, _ in self._ln_keep])
        bep = (FP * n)(*[(be.ctypes.data_as(FP) if be is not None else None) for _, be in self._ln_keep])
        h = C.c_void_p()
        _lib.check(lib.dspgn_decoder_create_ex(C.byref(spec), Wp, bp, gp, bep, device, C.byref(h)))
        self.handle = h

    def close(self):
        if getattr(self, "handle", None):
            _lib.load().dspgn_decoder_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
