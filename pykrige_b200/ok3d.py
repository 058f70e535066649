"""OrdinaryKriging3D with the H100 ``backend='cuda'`` execute() path.

API mirror of the reference class (src/pykrige/ok3d.py:198-932).
"""
import numpy as np

from . import core
from ._base import KrigeBase
from .core import _adjust_for_anisotropy, _make_variogram_parameter_list, _initialize_variogram_model

P_INV_TYPES = ("pinv", "pinvh")


class _Krige3DMixin:
    """Constructor plumbing shared by the two 3-D classes (ok3d.py:221-330, uk3d.py:239-340)."""

    _ndim = 3

    def _init_common_3d(self, x, y, z, val, variogram_model, variogram_parameters, variogram_function, nlags,
                        weight, anisotropy_scaling_y, anisotropy_scaling_z, anisotropy_angle_x,
                        anisotropy_angle_y, anisotropy_angle_z, verbose, enable_plotting, exact_values,
                        pseudo_inv, pseudo_inv_type):
        self.pseudo_inv = bool(pseudo_inv)
        self.pseudo_inv_type = str(pseudo_inv_type)
        if self.pseudo_inv_type not in P_INV_TYPES:
            raise ValueError("pseudo inv type not valid: " + str(pseudo_inv_type))
        if not isinstance(exact_values, bool):
            raise ValueError("exact_values has to be boolean True or False")
        self.exact_values = exact_values
        self.coordinates_type = "euclidean"

        def _dim_ok(model):
            from .compat_gstools import validate_gstools

            validate_gstools(model)
            if model.field_dim < 3:
                raise ValueError("GSTools: model dim is not 3")

        ov = self._select_variogram(variogram_model, variogram_function, _dim_ok)
        if "gstools" in ov:
            m = ov["gstools"]
            variogram_parameters = []
            anisotropy_scaling_y, anisotropy_scaling_z = m.pykrige_anis_y, m.pykrige_anis_z
            anisotropy_angle_x, anisotropy_angle_y, anisotropy_angle_z = (
                m.pykrige_angle_x, m.pykrige_angle_y, m.pykrige_angle_z)

        self.X_ORIG = np.atleast_1d(np.squeeze(np.array(x, copy=True, dtype=np.float64)))
        self.Y_ORIG = np.atleast_1d(np.squeeze(np.array(y, copy=True, dtype=np.float64)))
        self.Z_ORIG = np.atleast_1d(np.squeeze(np.array(z, copy=True, dtype=np.float64)))
        self.VALUES = np.atleast_1d(np.squeeze(np.array(val, copy=True, dtype=np.float64)))
        self.verbose = verbose
        self.enable_plotting = enable_plotting
        if self.enable_plotting and self.verbose:
            print("Plotting Enabled\n")

        self.XCENTER = (np.amax(self.X_ORIG) + np.amin(self.X_ORIG)) / 2.0
        self.YCENTER = (np.amax(self.Y_ORIG) + np.amin(self.Y_ORIG)) / 2.0
        self.ZCENTER = (np.amax(self.Z_ORIG) + np.amin(self.Z_ORIG)) / 2.0
        self.anisotropy_scaling_y = anisotropy_scaling_y
        self.anisotropy_scaling_z = anisotropy_scaling_z
        self.anisotropy_angle_x = anisotropy_angle_x
        self.anisotropy_angle_y = anisotropy_angle_y
        self.anisotropy_angle_z = anisotropy_angle_z
        if self.verbose:
            print("Adjusting data for anisotropy...")
        self._readjust()

        if self.verbose:
            print("Initializing variogram model...")
        vp_temp = _make_variogram_parameter_list(self.variogram_model, variogram_parameters)
        self.lags, self.semivariance, self.variogram_model_parameters = _initialize_variogram_model(
            np.vstack((self.X_ADJUSTED, self.Y_ADJUSTED, self.Z_ADJUSTED)).T,
            self.VALUES, self.variogram_model, vp_temp, self.variogram_function, nlags, weight, "euclidean", lazy=True,
        )
        if self.verbose:
            self._print_variogram()
        if self.enable_plotting:
            self.display_variogram_model()
        self._statistics_policy("lazy")

    def _readjust(self):
        self.X_ADJUSTED, self.Y_ADJUSTED, self.Z_ADJUSTED = _adjust_for_anisotropy(
            np.vstack((self.X_ORIG, self.Y_ORIG, self.Z_ORIG)).T,
            [self.XCENTER, self.YCENTER, self.ZCENTER],
            [self.anisotropy_scaling_y, self.anisotropy_scaling_z],
            [self.anisotropy_angle_x, self.anisotropy_angle_y, self.anisotropy_angle_z],
        ).T

    def _stats_inputs(self):
        return np.vstack((self.X_ADJUSTED, self.Y_ADJUSTED, self.Z_ADJUSTED)).T, self.VALUES

    def update_variogram_model(self, variogram_model, variogram_parameters=None, variogram_function=None,
                               nlags=6, weight=False, anisotropy_scaling_y=1.0, anisotropy_scaling_z=1.0,
                               anisotropy_angle_x=0.0, anisotropy_angle_y=0.0, anisotropy_angle_z=0.0):
        """Change the variogram model and/or its parameters (ok3d.py:354-520)."""

        def _dim_ok(model):
            from .compat_gstools import validate_gstools

            validate_gstools(model)
            if model.field_dim < 3:
                raise ValueError("GSTools: model dim is not 3")

        ov = self._select_variogram(variogram_model, variogram_function, _dim_ok)
        if "gstools" in ov:
            m = ov["gstools"]
            variogram_parameters = []
            anisotropy_scaling_y, anisotropy_scaling_z = m.pykrige_anis_y, m.pykrige_anis_z
            anisotropy_angle_x, anisotropy_angle_y, anisotropy_angle_z = (
                m.pykrige_angle_x, m.pykrige_angle_y, m.pykrige_angle_z)
        new = (anisotropy_scaling_y, anisotropy_scaling_z, anisotropy_angle_x, anisotropy_angle_y, anisotropy_angle_z)
        old = (self.anisotropy_scaling_y, self.anisotropy_scaling_z, self.anisotropy_angle_x,
               self.anisotropy_angle_y, self.anisotropy_angle_z)
        if new != old:
            if self.verbose:
                print("Adjusting data for anisotropy...")
            (self.anisotropy_scaling_y, self.anisotropy_scaling_z, self.anisotropy_angle_x,
             self.anisotropy_angle_y, self.anisotropy_angle_z) = new
            self._readjust()
        if self.verbose:
            print("Updating variogram mode...")
        vp_temp = _make_variogram_parameter_list(self.variogram_model, variogram_parameters)
        self.lags, self.semivariance, self.variogram_model_parameters = _initialize_variogram_model(
            np.vstack((self.X_ADJUSTED, self.Y_ADJUSTED, self.Z_ADJUSTED)).T,
            self.VALUES, self.variogram_model, vp_temp, self.variogram_function, nlags, weight, "euclidean", lazy=True,
        )
        if self.verbose:
            self._print_variogram()
        if self.enable_plotting:
            self.display_variogram_model()
        self._statistics_policy("lazy")

    def _data_arrays(self):
        Mt = core.anisotropy_matrix(
            3, [self.anisotropy_scaling_y, self.anisotropy_scaling_z],
            [self.anisotropy_angle_x, self.anisotropy_angle_y, self.anisotropy_angle_z])
        return (self.X_ORIG, self.Y_ORIG, self.Z_ORIG, self.VALUES,
                [self.XCENTER, self.YCENTER, self.ZCENTER], Mt)


class OrdinaryKriging3D(_Krige3DMixin, KrigeBase):
    """Three-dimensional ordinary kriging; arguments as in the reference docstring (ok3d.py:37-196)."""

    def __init__(self, x, y, z, val, variogram_model="linear", variogram_parameters=None, variogram_function=None,
                 nlags=6, weight=False, anisotropy_scaling_y=1.0, anisotropy_scaling_z=1.0, anisotropy_angle_x=0.0,
                 anisotropy_angle_y=0.0, anisotropy_angle_z=0.0, verbose=False, enable_plotting=False,
                 exact_values=True, pseudo_inv=False, pseudo_inv_type="pinv"):
        self._init_common_3d(x, y, z, val, variogram_model, variogram_parameters, variogram_function, nlags,
                             weight, anisotropy_scaling_y, anisotropy_scaling_z, anisotropy_angle_x,
                             anisotropy_angle_y, anisotropy_angle_z, verbose, enable_plotting, exact_values,
                             pseudo_inv, pseudo_inv_type)

    def execute(self, style, xpoints, ypoints, zpoints, mask=None, backend="cuda", n_closest_points=None,
                dtype="float64", n_gpus=None):
        """Calculates a kriged 3-D grid and the associated variance (ok3d.py:735-932); ``backend='cuda'``.
        Output shape (nz, ny, nx) for 'grid'/'masked', (n,) for 'points'."""
        if self.verbose:
            print("Executing Ordinary Kriging...\n")
        axes, sizes, flat_mask = self._prepare_points(style, (xpoints, ypoints, zpoints), mask)
        if n_closest_points is not None and n_closest_points <= 1:
            raise ValueError("n_closest_points has to be at least two!")
        self._check_backend(backend, "3D ordinary kriging")
        kvalues, sigmasq = self._run_cuda(style, axes, flat_mask, n_closest_points=n_closest_points, dtype=dtype,
                                          n_gpus=n_gpus)
        return self._shape_output(style, kvalues, sigmasq, sizes, flat_mask)
