"""numpy restatement of pycocotools 2.0.x's keypoint evaluation, the checker of ``centerpose_b200.coco_eval``.

Follows, statement for statement and in numpy's float64 arithmetic:
  * ``COCO.createIndex`` / ``getImgIds`` / ``getCatIds`` / ``getAnnIds`` / ``loadAnns`` (annotations grouped per image in
    file order; ``loadAnns`` looks ids up in a dict, so duplicate ids collapse onto the last annotation);
  * ``COCO.loadRes`` for a list of result dicts: the ``bbox`` branch when the first result has a non-empty bbox (what
    ``convert_eval_format`` writes: area = w * h), else the ``keypoints`` branch (area and bbox from the keypoints'
    extent); ids 1-based in results order; image ids outside the ground truth and empty results refused;
  * ``Params(iouType="keypoints")``;
  * ``COCOeval._prepare``, ``computeOks``, ``evaluateImg``, ``accumulate`` and ``summarize`` (``_summarizeKps``).

pycocotools is third-party; this module restates its published algorithm and is fed, as ``COCO.loadRes`` is by the
reference's ``dataset.run_eval``, with ``centerpose_b200.coco_format.convert_eval_format``'s output.
"""
from __future__ import annotations

import copy
from collections import defaultdict

import numpy as np


class Params:
    """``cocoeval.Params.setKpParams``."""

    def __init__(self):
        self.imgIds = []
        self.catIds = []
        self.iouThrs = np.linspace(.5, 0.95, int(np.round((0.95 - .5) / .05)) + 1, endpoint=True)
        self.recThrs = np.linspace(.0, 1.00, int(np.round((1.00 - .0) / .01)) + 1, endpoint=True)
        self.maxDets = [20]
        self.areaRng = [[0 ** 2, 1e5 ** 2], [32 ** 2, 96 ** 2], [96 ** 2, 1e5 ** 2]]
        self.areaRngLbl = ['all', 'medium', 'large']
        self.useCats = 1
        self.kpt_oks_sigmas = np.array([.26, .25, .25, .35, .35, .79, .79, .72, .72, .62, .62, 1.07, 1.07, .87, .87,
                                        .89, .89]) / 10.0
        self.iouType = 'keypoints'


class COCO:
    """The index ``COCOeval`` reads from a ground-truth or result set."""

    def __init__(self, dataset):
        self.dataset = dataset
        self.anns, self.cats, self.imgs = {}, {}, {}
        self.imgToAnns = defaultdict(list)
        for ann in dataset.get('annotations', []):
            self.imgToAnns[ann['image_id']].append(ann)
            self.anns[ann['id']] = ann
        for img in dataset.get('images', []):
            self.imgs[img['id']] = img
        for cat in dataset.get('categories', []):
            self.cats[cat['id']] = cat

    def getImgIds(self):
        return list(self.imgs.keys())

    def getCatIds(self):
        return [cat['id'] for cat in self.dataset.get('categories', [])]

    def getAnnIds(self, imgIds, catIds):
        lists = [self.imgToAnns[i] for i in imgIds if i in self.imgToAnns]
        anns = [a for lst in lists for a in lst]
        anns = anns if len(catIds) == 0 else [a for a in anns if a['category_id'] in catIds]
        return [a['id'] for a in anns]

    def loadAnns(self, ids):
        return [self.anns[i] for i in ids]

    def loadRes(self, anns):
        res = COCO({'images': list(self.dataset['images'])})
        anns = copy.deepcopy(anns)
        assert type(anns) == list, 'results in not an array of objects'
        ann_img_ids = [a['image_id'] for a in anns]
        assert set(ann_img_ids) == (set(ann_img_ids) & set(self.getImgIds())), \
            'Results do not correspond to current coco set'
        if 'bbox' in anns[0] and not anns[0]['bbox'] == []:
            res.dataset['categories'] = copy.deepcopy(self.dataset['categories'])
            for id, ann in enumerate(anns):
                bb = ann['bbox']
                ann['area'] = bb[2] * bb[3]
                ann['id'] = id + 1
                ann['iscrowd'] = 0
        elif 'keypoints' in anns[0]:
            res.dataset['categories'] = copy.deepcopy(self.dataset['categories'])
            for id, ann in enumerate(anns):
                s = ann['keypoints']
                x = s[0::3]
                y = s[1::3]
                x0, x1, y0, y1 = np.min(x), np.max(x), np.min(y), np.max(y)
                ann['area'] = (x1 - x0) * (y1 - y0)
                ann['id'] = id + 1
                ann['bbox'] = [x0, y0, x1 - x0, y1 - y0]
        else:
            raise NotImplementedError('only bbox or keypoints results')
        res.dataset['annotations'] = anns
        return COCO(res.dataset)


class COCOeval:
    """``COCOeval(cocoGt, cocoDt, "keypoints")``."""

    def __init__(self, cocoGt, cocoDt):
        self.cocoGt, self.cocoDt = cocoGt, cocoDt
        self.params = Params()
        self.params.imgIds = sorted(cocoGt.getImgIds())
        self.params.catIds = sorted(cocoGt.getCatIds())
        self.eval = {}
        self.stats = []

    def _prepare(self):
        p = self.params
        gts = self.cocoGt.loadAnns(self.cocoGt.getAnnIds(imgIds=p.imgIds, catIds=p.catIds))
        dts = self.cocoDt.loadAnns(self.cocoDt.getAnnIds(imgIds=p.imgIds, catIds=p.catIds))
        for gt in gts:
            gt['ignore'] = gt['ignore'] if 'ignore' in gt else 0
            gt['ignore'] = 'iscrowd' in gt and gt['iscrowd']
            gt['ignore'] = (gt['num_keypoints'] == 0) or gt['ignore']
        self._gts = defaultdict(list)
        self._dts = defaultdict(list)
        for gt in gts:
            self._gts[gt['image_id'], gt['category_id']].append(gt)
        for dt in dts:
            self._dts[dt['image_id'], dt['category_id']].append(dt)

    def evaluate(self):
        p = self.params
        p.imgIds = list(np.unique(p.imgIds))
        p.catIds = list(np.unique(p.catIds))
        p.maxDets = sorted(p.maxDets)
        self._prepare()
        self.ious = {(i, c): self.computeOks(i, c) for i in p.imgIds for c in p.catIds}
        maxDet = p.maxDets[-1]
        self.evalImgs = [self.evaluateImg(i, c, a, maxDet) for c in p.catIds for a in p.areaRng for i in p.imgIds]
        self._paramsEval = copy.deepcopy(self.params)

    def computeOks(self, imgId, catId):
        p = self.params
        gts = self._gts[imgId, catId]
        dts = self._dts[imgId, catId]
        inds = np.argsort([-d['score'] for d in dts], kind='mergesort')
        dts = [dts[i] for i in inds]
        if len(dts) > p.maxDets[-1]:
            dts = dts[0:p.maxDets[-1]]
        if len(gts) == 0 or len(dts) == 0:
            return []
        ious = np.zeros((len(dts), len(gts)))
        sigmas = p.kpt_oks_sigmas
        vars = (sigmas * 2) ** 2
        k = len(sigmas)
        for j, gt in enumerate(gts):
            g = np.array(gt['keypoints'])
            xg = g[0::3]; yg = g[1::3]; vg = g[2::3]
            k1 = np.count_nonzero(vg > 0)
            bb = gt['bbox']
            x0 = bb[0] - bb[2]; x1 = bb[0] + bb[2] * 2
            y0 = bb[1] - bb[3]; y1 = bb[1] + bb[3] * 2
            for i, dt in enumerate(dts):
                d = np.array(dt['keypoints'])
                xd = d[0::3]; yd = d[1::3]
                if k1 > 0:
                    dx = xd - xg
                    dy = yd - yg
                else:
                    z = np.zeros((k))
                    dx = np.max((z, x0 - xd), axis=0) + np.max((z, xd - x1), axis=0)
                    dy = np.max((z, y0 - yd), axis=0) + np.max((z, yd - y1), axis=0)
                e = (dx ** 2 + dy ** 2) / vars / (gt['area'] + np.spacing(1)) / 2
                if k1 > 0:
                    e = e[vg > 0]
                ious[i, j] = np.sum(np.exp(-e)) / e.shape[0]
        return ious

    def evaluateImg(self, imgId, catId, aRng, maxDet):
        p = self.params
        gt = self._gts[imgId, catId]
        dt = self._dts[imgId, catId]
        if len(gt) == 0 and len(dt) == 0:
            return None
        for g in gt:
            g['_ignore'] = 1 if g['ignore'] or (g['area'] < aRng[0] or g['area'] > aRng[1]) else 0
        gtind = np.argsort([g['_ignore'] for g in gt], kind='mergesort')
        gt = [gt[i] for i in gtind]
        dtind = np.argsort([-d['score'] for d in dt], kind='mergesort')
        dt = [dt[i] for i in dtind[0:maxDet]]
        iscrowd = [int(o['iscrowd']) for o in gt]
        ious = self.ious[imgId, catId][:, gtind] if len(self.ious[imgId, catId]) > 0 else self.ious[imgId, catId]
        T = len(p.iouThrs); G = len(gt); D = len(dt)
        gtm = np.zeros((T, G))
        dtm = np.zeros((T, D))
        gtIg = np.array([g['_ignore'] for g in gt])
        dtIg = np.zeros((T, D))
        if not len(ious) == 0:
            for tind, t in enumerate(p.iouThrs):
                for dind, d in enumerate(dt):
                    iou = min([t, 1 - 1e-10])
                    m = -1
                    for gind, g in enumerate(gt):
                        if gtm[tind, gind] > 0 and not iscrowd[gind]:
                            continue
                        if m > -1 and gtIg[m] == 0 and gtIg[gind] == 1:
                            break
                        if ious[dind, gind] < iou:
                            continue
                        iou = ious[dind, gind]
                        m = gind
                    if m == -1:
                        continue
                    dtIg[tind, dind] = gtIg[m]
                    dtm[tind, dind] = gt[m]['id']
                    gtm[tind, m] = d['id']
        a = np.array([d['area'] < aRng[0] or d['area'] > aRng[1] for d in dt]).reshape((1, len(dt)))
        dtIg = np.logical_or(dtIg, np.logical_and(dtm == 0, np.repeat(a, T, 0)))
        return {'image_id': imgId, 'category_id': catId, 'aRng': aRng, 'maxDet': maxDet,
                'dtIds': [d['id'] for d in dt], 'gtIds': [g['id'] for g in gt],
                'dtMatches': dtm, 'gtMatches': gtm, 'dtScores': [d['score'] for d in dt],
                'gtIgnore': gtIg, 'dtIgnore': dtIg}

    def accumulate(self):
        p = self.params
        T = len(p.iouThrs); R = len(p.recThrs); K = len(p.catIds); A = len(p.areaRng); M = len(p.maxDets)
        precision = -np.ones((T, R, K, A, M))
        recall = -np.ones((T, K, A, M))
        scores = -np.ones((T, R, K, A, M))
        _pe = self._paramsEval
        setK = set(_pe.catIds); setA = set(map(tuple, _pe.areaRng)); setM = set(_pe.maxDets); setI = set(_pe.imgIds)
        k_list = [n for n, k in enumerate(p.catIds) if k in setK]
        m_list = [m for n, m in enumerate(p.maxDets) if m in setM]
        a_list = [n for n, a in enumerate(map(lambda x: tuple(x), p.areaRng)) if a in setA]
        i_list = [n for n, i in enumerate(p.imgIds) if i in setI]
        I0 = len(_pe.imgIds); A0 = len(_pe.areaRng)
        for k, k0 in enumerate(k_list):
            Nk = k0 * A0 * I0
            for a, a0 in enumerate(a_list):
                Na = a0 * I0
                for m, maxDet in enumerate(m_list):
                    E = [self.evalImgs[Nk + Na + i] for i in i_list]
                    E = [e for e in E if e is not None]
                    if len(E) == 0:
                        continue
                    dtScores = np.concatenate([e['dtScores'][0:maxDet] for e in E])
                    inds = np.argsort(-dtScores, kind='mergesort')
                    dtScoresSorted = dtScores[inds]
                    dtm = np.concatenate([e['dtMatches'][:, 0:maxDet] for e in E], axis=1)[:, inds]
                    dtIg = np.concatenate([e['dtIgnore'][:, 0:maxDet] for e in E], axis=1)[:, inds]
                    gtIg = np.concatenate([e['gtIgnore'] for e in E])
                    npig = np.count_nonzero(gtIg == 0)
                    if npig == 0:
                        continue
                    tps = np.logical_and(dtm, np.logical_not(dtIg))
                    fps = np.logical_and(np.logical_not(dtm), np.logical_not(dtIg))
                    tp_sum = np.cumsum(tps, axis=1).astype(dtype=np.float64)
                    fp_sum = np.cumsum(fps, axis=1).astype(dtype=np.float64)
                    for t, (tp, fp) in enumerate(zip(tp_sum, fp_sum)):
                        tp = np.array(tp)
                        fp = np.array(fp)
                        nd = len(tp)
                        rc = tp / npig
                        pr = tp / (fp + tp + np.spacing(1))
                        q = np.zeros((R,))
                        ss = np.zeros((R,))
                        recall[t, k, a, m] = rc[-1] if nd else 0
                        pr = pr.tolist(); q = q.tolist()
                        for i in range(nd - 1, 0, -1):
                            if pr[i] > pr[i - 1]:
                                pr[i - 1] = pr[i]
                        inds = np.searchsorted(rc, p.recThrs, side='left')
                        try:
                            for ri, pi in enumerate(inds):
                                q[ri] = pr[pi]
                                ss[ri] = dtScoresSorted[pi]
                        except IndexError:
                            pass
                        precision[t, :, k, a, m] = np.array(q)
                        scores[t, :, k, a, m] = np.array(ss)
        self.eval = {'params': p, 'counts': [T, R, K, A, M], 'precision': precision, 'recall': recall,
                     'scores': scores}

    def summarize(self, out=print):
        """``_summarizeKps``: the ten stats; each line goes to ``out``."""
        p = self.params

        def _summarize(ap=1, iouThr=None, areaRng='all', maxDets=100):
            iStr = ' {:<18} {} @[ IoU={:<9} | area={:>6s} | maxDets={:>3d} ] = {:0.3f}'
            titleStr = 'Average Precision' if ap == 1 else 'Average Recall'
            typeStr = '(AP)' if ap == 1 else '(AR)'
            iouStr = '{:0.2f}:{:0.2f}'.format(p.iouThrs[0], p.iouThrs[-1]) if iouThr is None else '{:0.2f}'.format(iouThr)
            aind = [i for i, aRng in enumerate(p.areaRngLbl) if aRng == areaRng]
            mind = [i for i, mDet in enumerate(p.maxDets) if mDet == maxDets]
            if ap == 1:
                s = self.eval['precision']
                if iouThr is not None:
                    s = s[np.where(iouThr == p.iouThrs)[0]]
                s = s[:, :, :, aind, mind]
            else:
                s = self.eval['recall']
                if iouThr is not None:
                    s = s[np.where(iouThr == p.iouThrs)[0]]
                s = s[:, :, aind, mind]
            mean_s = -1 if len(s[s > -1]) == 0 else np.mean(s[s > -1])
            out(iStr.format(titleStr, typeStr, iouStr, areaRng, maxDets, mean_s))
            return mean_s

        stats = np.zeros((10,))
        stats[0] = _summarize(1, maxDets=20)
        stats[1] = _summarize(1, maxDets=20, iouThr=.5)
        stats[2] = _summarize(1, maxDets=20, iouThr=.75)
        stats[3] = _summarize(1, maxDets=20, areaRng='medium')
        stats[4] = _summarize(1, maxDets=20, areaRng='large')
        stats[5] = _summarize(0, maxDets=20)
        stats[6] = _summarize(0, maxDets=20, iouThr=.5)
        stats[7] = _summarize(0, maxDets=20, iouThr=.75)
        stats[8] = _summarize(0, maxDets=20, areaRng='medium')
        stats[9] = _summarize(0, maxDets=20, areaRng='large')
        self.stats = stats
        return stats


def evaluate(gt_dataset, detections, img_ids=None, out=print):
    """``COCOeval(gt, gt.loadRes(detections), "keypoints")``'s evaluate / accumulate / summarize on a ground-truth
    dict and a list of result dicts.  The ground truth is copied (``_prepare`` writes into its annotations).
    Returns the ``COCOeval``: ``.eval`` and ``.stats`` filled, ``.lines`` the summary lines."""
    gt = COCO(copy.deepcopy(gt_dataset))
    E = COCOeval(gt, gt.loadRes(detections))
    if img_ids is not None:
        E.params.imgIds = list(img_ids)
    E.evaluate()
    E.accumulate()
    E.lines = []
    E.summarize(out=lambda s: (E.lines.append(s), out and out(s)))
    return E
