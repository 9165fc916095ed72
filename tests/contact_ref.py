"""numpy restatement of the reference's contact queries (robosuite v1.5.2, utils/sim_utils.py check_contact / get_contacts,
manipulation_env.py _check_grasp; recalled, see robosuite_b200/envs/contacts.py), one environment at a time, looping over the
contact list data.contact[:ncon] as the reference does.  Geoms are compared by id (the reference compares names, which is the same
for the named geoms these tests query)."""
import numpy as np


def _ids(model, geoms):
    gn = model.names["geom"]
    if isinstance(geoms, (str, int, np.integer)):
        geoms = [geoms]
    return {gn.index(g) if isinstance(g, str) else int(g) for g in geoms}


def _pairs(ncon, geom):
    return [(int(a), int(b)) for a, b in np.asarray(geom)[: int(ncon)]]


def check_contact(model, ncon, geom, geoms_1, geoms_2=None):
    g1s = _ids(model, geoms_1)
    g2s = None if geoms_2 is None else _ids(model, geoms_2)
    for c1, c2 in _pairs(ncon, geom):
        c1_in_g1 = c1 in g1s
        c2_in_g2 = c2 in g2s if g2s is not None else True
        c2_in_g1 = c2 in g1s
        c1_in_g2 = c1 in g2s if g2s is not None else True
        if (c1_in_g1 and c2_in_g2) or (c1_in_g2 and c2_in_g1):
            return True
    return False


def get_contacts(model, ncon, geom, geoms):
    """the reference's geom set, as a bool [ngeom] mask"""
    s = _ids(model, geoms)
    out = np.zeros(int(model.ngeom), dtype=bool)
    for c1, c2 in _pairs(ncon, geom):
        if c1 in s and c2 not in s:
            out[c2] = True
        elif c2 in s and c1 not in s:
            out[c1] = True
    return out


def check_grasp(model, ncon, geom, groups, object_geoms):
    return all(check_contact(model, ncon, geom, g, object_geoms) for g in groups)
