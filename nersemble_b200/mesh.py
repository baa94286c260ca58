"""Triangle-mesh results of NeRSembleNGPModel.extract_mesh / extract_mesh_sequence (ops.extract_mesh /
ops.extract_mesh_sequence) and their PLY export (numpy only)."""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Sequence

import numpy as np


@dataclass
class Mesh:
    vertices: np.ndarray                    # float32 [V, 3], world space
    faces: np.ndarray                       # int32 [F, 3], counter-clockwise seen from outside
    normals: Optional[np.ndarray] = None    # float32 [V, 3] unit (zero where undefined)
    colours: Optional[np.ndarray] = None    # float32 [V, 3] in [0, 1]

    @staticmethod
    def from_tensors(out: dict) -> "Mesh":
        """From the dict of ops.extract_mesh (device tensors)."""
        get = lambda k, dt: None if out.get(k) is None else out[k].detach().cpu().numpy().astype(dt)
        return Mesh(get("vertices", np.float32), get("faces", np.int32), get("normals", np.float32), get("colours", np.float32))

    def save_ply(self, path: str) -> None:
        """Binary little-endian PLY: x y z (+ nx ny nz) as float, red green blue as uchar, faces as a uchar-counted int
        list.  Colours are rounded from [0, 1] to 0..255."""
        V, F = len(self.vertices), len(self.faces)
        fields = [("x", "<f4"), ("y", "<f4"), ("z", "<f4")]
        if self.normals is not None:
            fields += [("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4")]
        if self.colours is not None:
            fields += [("red", "u1"), ("green", "u1"), ("blue", "u1")]
        vert = np.empty(V, dtype=fields)
        for k, name in enumerate("xyz"):
            vert[name] = self.vertices[:, k]
        if self.normals is not None:
            for k, name in enumerate(("nx", "ny", "nz")):
                vert[name] = self.normals[:, k]
        if self.colours is not None:
            rgb = np.clip(np.rint(np.asarray(self.colours, dtype=np.float64) * 255.0), 0, 255).astype(np.uint8)
            for k, name in enumerate(("red", "green", "blue")):
                vert[name] = rgb[:, k]
        face = np.empty(F, dtype=[("n", "u1"), ("v", "<i4", (3,))])
        face["n"] = 3
        face["v"] = self.faces
        ply_type = {"<f4": "float", "u1": "uchar"}
        head = ["ply", "format binary_little_endian 1.0", f"element vertex {V}"]
        head += [f"property {ply_type[t]} {name}" for name, t in fields]
        head += [f"element face {F}", "property list uchar int vertex_indices", "end_header"]
        with open(path, "wb") as f:
            f.write(("\n".join(head) + "\n").encode("ascii"))
            f.write(vert.tobytes())
            f.write(face.tobytes())

    @staticmethod
    def load_ply(path: str) -> "Mesh":
        """Reads what save_ply writes (binary little-endian, triangle faces); colours come back as uchar / 255."""
        with open(path, "rb") as f:
            data = f.read()
        end = data.index(b"end_header\n") + len(b"end_header\n")
        lines = data[:end].decode("ascii").splitlines()
        if lines[0] != "ply" or lines[1] != "format binary_little_endian 1.0":
            raise ValueError(f"{path}: not a binary little-endian PLY")
        fields, V, F, elem = [], 0, 0, None
        for ln in lines[2:]:
            w = ln.split()
            if w[0] == "element":
                elem = w[1]
                if elem == "vertex":
                    V = int(w[2])
                elif elem == "face":
                    F = int(w[2])
            elif w[0] == "property" and elem == "vertex":
                fields.append((w[2], {"float": "<f4", "uchar": "u1"}[w[1]]))
        vert = np.frombuffer(data, dtype=fields, count=V, offset=end)
        face = np.frombuffer(data, dtype=[("n", "u1"), ("v", "<i4", (3,))], count=F, offset=end + vert.nbytes)
        if F and (face["n"] != 3).any():
            raise ValueError(f"{path}: only triangle faces are supported")
        names = [n for n, _ in fields]
        stack = lambda keys, dt: np.stack([vert[k] for k in keys], -1).astype(dt) if all(k in names for k in keys) else None
        rgb = stack(("red", "green", "blue"), np.float32)
        return Mesh(stack("xyz", np.float32), np.ascontiguousarray(face["v"], dtype=np.int32),
                    stack(("nx", "ny", "nz"), np.float32), None if rgb is None else rgb / 255.0)


@dataclass
class MeshSequence:
    """One connectivity for every frame: the reference frame's mesh with its vertices tracked along the deformation
    field.  converged[i, v] says whether vertex v's track to frame i converged; sigma[i, v] is the density at the tracked
    vertex (near the extraction level where the deformation alone moved the surface, away from it where the hash
    ensemble's blend moved it)."""
    faces: np.ndarray                       # int32 [F, 3], shared by every frame
    vertices: np.ndarray                    # float32 [K, V, 3], world space
    timesteps: List[int]                    # the frames' timesteps
    converged: np.ndarray                   # bool [K, V]
    sigma: np.ndarray                       # float32 [K, V]
    normals: Optional[np.ndarray] = None    # float32 [K, V, 3]
    colours: Optional[np.ndarray] = None    # float32 [K, V, 3]

    @staticmethod
    def from_tensors(out: dict, timesteps: Sequence[int]) -> "MeshSequence":
        """From the dict of ops.extract_mesh_sequence (device tensors)."""
        get = lambda k, dt: None if out.get(k) is None else out[k].detach().cpu().numpy().astype(dt)
        return MeshSequence(get("faces", np.int32), get("vertices", np.float32), [int(t) for t in timesteps],
                            get("converged", bool), get("sigma", np.float32), get("normals", np.float32),
                            get("colours", np.float32))

    def __len__(self) -> int:
        return len(self.timesteps)

    def frame(self, i: int) -> Mesh:
        """Frame i (index into timesteps) as a Mesh."""
        pick = lambda a: None if a is None else a[i]
        return Mesh(self.vertices[i], self.faces, pick(self.normals), pick(self.colours))

    def save_ply(self, pattern: str) -> List[str]:
        """One PLY per frame through Mesh.save_ply; pattern.format(timestep) names each file (e.g. "head_{:03d}.ply").
        Returns the paths."""
        paths = []
        for i, t in enumerate(self.timesteps):
            path = pattern.format(t)
            if path in paths:
                raise ValueError(f"the pattern {pattern!r} gives the same file for two frames")
            self.frame(i).save_ply(path)
            paths.append(path)
        return paths
